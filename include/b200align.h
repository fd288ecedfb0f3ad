/*
 * b200align.h -- C ABI of libb200align.so: the drop-in boundary for the
 * `bio::alignment::pairwise` hot path of rust-bio 4.0.1, rebuilt H100-native.
 *
 * The reference has no FFI for this path: its boundary is the Rust method
 * surface (reference src/alignment/pairwise/mod.rs):
 *     Scoring<F>                       mod.rs:238-429
 *     Aligner::with_capacity / ...     mod.rs:495-583
 *     Aligner::custom                  mod.rs:591-922
 *     Aligner::global                  mod.rs:925-951
 *     Aligner::semiglobal              mod.rs:954-983
 *     Aligner::local                   mod.rs:986-1015
 *     banded::Aligner::*               banded.rs:150-401, 872-1004
 * A per-pair call cannot feed a GPU, so every entry point here is the BATCH
 * form of one of those methods; a single-pair call is a batch of one.  The
 * Rust shim (rust_bio_b200/rust/src/lib.rs) and the Python mirror
 * (rust_bio_b200/pairwise.py) bind exactly these symbols.
 *
 * Conventions
 *   - plain C, no exceptions / unwinding across the boundary;
 *   - every function returns 0 on success or a negative B2A_E_* code;
 *     b2a_last_error() gives the text for the calling engine;
 *   - an engine handle is bound to ONE CUDA device and may be used by one
 *     host thread at a time (the reference's `&mut self` contract,
 *     mod.rs:591,925,954,986);
 *   - there is NO CPU fallback: every align call fails with
 *     B2A_E_NO_DEVICE if the CUDA device cannot be used.
 */
#ifndef B200ALIGN_H_
#define B200ALIGN_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* pairwise::MIN_SCORE (mod.rs:174) */
#define B2A_MIN_SCORE (-858993459)

/* banded::MAX_CELLS (banded.rs:104) */
#define B2A_BANDED_MAX_CELLS 5000000ull

/* AlignmentMode, in bio-types variant order (used at mod.rs:920,942,971,1003) */
enum {
  B2A_MODE_CUSTOM = 0,     /* Aligner::custom      mod.rs:591 */
  B2A_MODE_GLOBAL = 1,     /* Aligner::global      mod.rs:925 */
  B2A_MODE_SEMIGLOBAL = 2, /* Aligner::semiglobal  mod.rs:954 */
  B2A_MODE_LOCAL = 3       /* Aligner::local       mod.rs:986 */
};

/* AlignmentOperation codes (bio-types variant order; pushed at mod.rs:860-900) */
enum {
  B2A_OP_MATCH = 0,
  B2A_OP_SUBST = 1,
  B2A_OP_DEL = 2,
  B2A_OP_INS = 3,
  B2A_OP_XCLIP = 4, /* length is in clip_len, in order of appearance */
  B2A_OP_YCLIP = 5
};

/* error codes */
enum {
  B2A_OK = 0,
  B2A_E_INVALID = -1,     /* bad argument (the reference would panic: mod.rs:517-518,554-571) */
  B2A_E_NO_DEVICE = -2,   /* CUDA device / driver unusable: no CPU fallback exists */
  B2A_E_CUDA = -3,        /* a CUDA runtime call failed; see b2a_last_error */
  B2A_E_RANGE = -4,       /* scores/lengths would overflow i32 in the reference recurrence */
  B2A_E_CAPACITY = -5,    /* caller's ops buffer too small */
  B2A_E_STATE = -6,       /* stage/run/fetch called out of order */
  B2A_E_UNSUPPORTED = -7  /* a forced fill shape that cannot stage the batch's sequences on chip, or one pair whose
                             traceback alone exceeds the traceback budget (the score-only calls align it) */
};

/* Scoring<F> (mod.rs:238-247).  `table`, when non-NULL, is the host-tabulated
 * MatchFunc: 256x256 row-major, table[a*256+b] = match_fn.score(a, b)
 * (mod.rs:177-228); only entries for symbols present in the batch are read.
 * When NULL, MatchParams semantics apply (mod.rs:208-217).
 * has_match_scores/match_score mirror `match_scores: Option<(i32,i32)>`
 * (mod.rs:242), which only banded::Band::create consults (banded.rs:1315-1318). */
typedef struct b2a_scoring {
  int32_t gap_open;
  int32_t gap_extend;
  int32_t xclip_prefix;
  int32_t xclip_suffix;
  int32_t yclip_prefix;
  int32_t yclip_suffix;
  int32_t match_score;
  int32_t mismatch_score;
  int32_t has_match_scores;
  const int32_t* table;
  /* Symbols for which `table` is valid (e.g. "A-Z*" for bio::scores matrices).
   * NULL with a non-NULL table: the engine scans the batch for the symbols
   * present (slower).  That scan is one flat pass over all of seq_blob, so
   * bytes between sequences (padding) count as present: their table entries
   * take part in the |score| <= 2^27 check and the score bound.  Pass the
   * alphabet when such bytes have large or undefined entries.
   * A sequence byte outside the alphabet is B2A_E_INVALID
   * (bio::scores::lookup would index out of bounds, scores/mod.rs:22-35). */
  const uint8_t* alphabet;
  uint32_t alphabet_len;
} b2a_scoring;

/* A batch of (x, y) pairs: TextSlice arguments of the align methods. */
typedef struct b2a_pairs {
  const uint8_t* seq_blob;  /* all sequences, any layout */
  const uint64_t* x_off;    /* [n_pairs] byte offset of x in seq_blob */
  const uint32_t* x_len;    /* [n_pairs] m */
  const uint64_t* y_off;    /* [n_pairs] */
  const uint32_t* y_len;    /* [n_pairs] n */
  uint64_t blob_bytes;
  uint64_t n_pairs;
} b2a_pairs;

/* Caller-allocated host outputs == the fields of bio_types Alignment
 * (built at mod.rs:911-921); xlen/ylen/mode are known to the caller. */
typedef struct b2a_results {
  int32_t* score;      /* [n_pairs] */
  uint32_t* xstart;    /* [n_pairs] */
  uint32_t* xend;      /* [n_pairs] */
  uint32_t* ystart;    /* [n_pairs] */
  uint32_t* yend;      /* [n_pairs] */
  uint64_t* ops_off;   /* [n_pairs+1] prefix offsets into ops */
  uint8_t* ops;        /* [ops_capacity] B2A_OP_* codes, alignment order */
  uint64_t ops_capacity;
  uint32_t* clip_len;  /* [4*n_pairs] lengths of the Xclip/Yclip ops of a pair, in order of appearance */
  /* [n_pairs] B2A_PAIR_* per pair, or NULL.  The reference fails per CALL: a pair on which it would panic
   * (mod.rs:905 "Dint expect this!", banded.rs walk on a corrupt cell, an asserting caller-supplied match list)
   * or never return takes only that pair down.  With status == NULL such a pair fails the whole batch
   * (B2A_E_RANGE / B2A_E_INVALID / B2A_E_CAPACITY); with a status array the batch succeeds, the pair's status is
   * non-zero and its other outputs are score = B2A_MIN_SCORE, no ops. */
  uint32_t* status;
} b2a_results;

enum {
  B2A_PAIR_OK = 0,
  B2A_PAIR_PANIC = 1,        /* the reference panics (or loops forever) on this pair */
  B2A_PAIR_CAPACITY = 2,     /* banded: more k-mer matches than the engine's per-pair limit (2^22) */
  B2A_PAIR_INVALID_HINT = 4  /* banded: caller-supplied matches/path the reference asserts on */
};

typedef struct b2a_stats {
  uint64_t cells;          /* sum of DP cells (m*n, or Band::num_cells for banded) */
  uint64_t h2d_bytes;
  uint64_t d2h_bytes;
  uint64_t traceback_bytes; /* traceback bit-vector bytes the fill kernel stores (a recomputed pair: what its refills
                                store, window by window) */
  float pack_ms;           /* K0 */
  float fill_ms;           /* K1 (or K3) */
  float walk_ms;           /* K2 epilogue + traceback walk (+ ops compaction) */
  float band_ms;           /* K4 (banded only) */
  uint32_t kernel_launches;
  uint32_t waves;          /* sub-batches the traceback budget forced */
  uint32_t fill_lanes_per_pair; /* G of the fill kernel variant used */
  uint32_t fill_rows_per_lane;  /* R */
} b2a_stats;

typedef struct b2a_engine b2a_engine;

/* lifecycle */
int32_t b2a_engine_create(b2a_engine** out, int32_t device_id);
int32_t b2a_engine_destroy(b2a_engine* e);
const char* b2a_last_error(const b2a_engine* e);
const char* b2a_version(void);

/* Run all engine work on this cudaStream_t (default: an engine-owned stream). */
int32_t b2a_engine_set_stream(b2a_engine* e, void* cuda_stream);
/* Upper bound (bytes) on device scratch for traceback bit-vectors; larger
 * batches are processed in waves. 0 = default (60% of free HBM).  With the warp-per-pair shape a block holds fewer
 * than 32 pairs when that keeps it within the budget, so waves can close between long pairs; a single pair whose
 * traceback alone is above the budget is B2A_E_UNSUPPORTED before anything is allocated, unless the traceback
 * recompute knob below is on. */
int32_t b2a_engine_set_traceback_budget(b2a_engine* e, uint64_t bytes);
/* on = 1: a warp-per-pair pair whose traceback alone is above the budget is aligned anyway, by recomputation: one
 * extra score-only fill checkpoints the strip boundary every W = floor(budget / strip bytes) strips, and the traceback
 * is refilled one window of W strips at a time as the walk reaches it (windows the walk jumps over are never filled).
 * Results are bit-identical to a budget that holds the pair.  Such a batch costs at least one more fill and a host
 * round trip per window.  A budget below one strip's traceback of the pair (K * TBW * 512 bytes) is still
 * B2A_E_UNSUPPORTED.  on = 0 (the default) keeps the refusal.  The chunk pipeline's engines inherit the setting. */
int32_t b2a_engine_set_traceback_recompute(b2a_engine* e, int32_t on);
/* Of the last b2a_align_batch / b2a_batch_stage + run: the pairs whose traceback was recomputed, their windows, and the
 * windows actually refilled (a measurement aid; any pointer may be NULL). */
int32_t b2a_engine_last_recompute(const b2a_engine* e, uint64_t* pairs, uint64_t* windows, uint64_t* windows_filled);
/* Force the fill-kernel shape (lanes per pair G in {1,2,4,8,32}, rows per
 * lane R in {8,16,20}: the built pairs are 1x8 1x16 1x20 2x16 2x20 4x16 8x16 8x20 32x8 32x16); 0,0 = automatic.
 * The shapes with several pairs per warp stage whole sequences in shared memory: forced, a batch they cannot stage
 * is B2A_E_UNSUPPORTED (the automatic choice falls back to the warp-per-pair shape).  32x8 and 32x16 stage one strip
 * of x and read y from device memory: they take any length up to 2^24. */
int32_t b2a_engine_set_tuning(b2a_engine* e, int32_t lanes_per_pair, int32_t rows_per_lane);

/* The alphabet the last stage used: the caller's, or the byte values the engine found in the batch when
 * b2a_scoring.alphabet was NULL (symbols[256], ascending).  A caller that cuts one batch into pieces can hand the
 * first piece's alphabet to the others (b2a_scoring.alphabet) and spare them the discovery pass and its
 * synchronisation; a piece holding a byte outside it fails with B2A_E_INVALID and is redone without. */
int32_t b2a_engine_last_alphabet(const b2a_engine* e, uint8_t* symbols, uint32_t* n_symbols);

/* K2 (row m, last-column fix-ups, traceback walk) runs one lane per pair (1) or one warp per pair (2);
 * 0 = automatic: warp per pair for waves of up to 16,384 pairs.  Results are identical either way. */
int32_t b2a_engine_set_walk(b2a_engine* e, int32_t mode);

/* b2a_align_batch cuts batches of >= 262,144 pairs into `chunks` pieces that alternate between two
 * internal engines, so one chunk's copies and host planning overlap the other's kernels.
 * chunks < 2 disables the pipeline (default 5, relative sizes 1,3,6,6,3). Results are identical either way. */
int32_t b2a_engine_set_pipeline(b2a_engine* e, int32_t chunks);

/* One-call form: Aligner::{custom,global,semiglobal,local} over a batch with
 * HOST inputs and HOST outputs (copies inside). mode = B2A_MODE_*. */
int32_t b2a_align_batch(b2a_engine* e, int32_t mode, const b2a_scoring* scoring,
                        const b2a_pairs* pairs, b2a_results* results, b2a_stats* stats);

/* Aligner::{custom,global,semiglobal,local} reduced to Alignment.score / xend / yend: no traceback is stored or walked.
 * For each pair, score, xend and yend are what b2a_align_batch returns; xstart, ystart and the ops are not computed
 * (they come out of the prefix end of the traceback walk).  The fill keeps no traceback, so waves close on the rest of
 * the per-wave scratch (boundary rows, row trackers, row m) against the traceback budget, and K2 walks only along
 * row m and column n: once the walk enters a cell with i < m and j < n, xend and yend are final.
 *   stage_scores: as b2a_batch_stage; b2a_batch_run then runs the score-only batch.
 *   b2a_batch_fetch on it fills score, xend, yend and status; xstart, ystart, ops, ops_off and clip_len must be NULL
 *   (else B2A_E_INVALID).  b2a_batch_records*, b2a_batch_compact* and b2a_gathered_fetch return B2A_E_STATE.
 *   b2a_align_batch_scores is single-shot at every size (no chunk pipeline).
 * A forced fill shape (b2a_engine_set_tuning) other than 1x16, 8x16, 8x20, 32x8 or 32x16 is B2A_E_UNSUPPORTED.
 * status: a pair whose walk would panic or never end while still on row m / column n is B2A_PAIR_PANIC, as with
 * b2a_align_batch.  A panic only the interior walk would meet (mod.rs:905) cannot be seen without the traceback:
 * such a pair reports its score.
 * The banded aligner's score-only form, under the same rule, is b2a_align_batch_banded_scores (below). */
int32_t b2a_batch_stage_scores(b2a_engine* e, int32_t mode, const b2a_scoring* scoring, const b2a_pairs* pairs);
int32_t b2a_align_batch_scores(b2a_engine* e, int32_t mode, const b2a_scoring* scoring, const b2a_pairs* pairs,
                               b2a_results* results, b2a_stats* stats);

/* Packed input (SURVEY 8f rank 2): the sequences as bio::data_structures::bitenc::BitEnc storage
 * (src/data_structures/bitenc.rs:50-56: 32-bit blocks, `width` bits per symbol, 32 - 32 % width usable bits per
 * block; symbol i sits at bit (i*width) % usable of block (i*width) / usable, bitenc.rs:319-338), holding the ranks
 * alphabets::RankTransform::transform yields (src/alphabets/mod.rs:220-283).  x_block / y_block are block indices
 * into `blocks`.  The packed blocks are what crosses PCIe (width 2: a quarter of the bytes); scores are those of
 * `scoring` applied to the RANKS: MatchParams by equality, `table[a*256+b]` indexed by rank. */
typedef struct b2a_packed_pairs {
  const uint32_t* blocks;   /* all BitEnc storages, concatenated */
  const uint64_t* x_block;  /* [n_pairs] first block of x */
  const uint32_t* x_len;    /* [n_pairs] symbols (BitEnc::nr_symbols) */
  const uint64_t* y_block;
  const uint32_t* y_len;
  uint64_t n_blocks;
  uint64_t n_pairs;
  uint32_t width;           /* BitEnc::new(width), 1..8 */
} b2a_packed_pairs;
int32_t b2a_align_batch_packed(b2a_engine* e, int32_t mode, const b2a_scoring* scoring,
                               const b2a_packed_pairs* pairs, b2a_results* results, b2a_stats* stats);
int32_t b2a_align_batch_banded_packed(b2a_engine* e, int32_t mode, const b2a_scoring* scoring, uint32_t k, uint32_t w,
                                      const b2a_packed_pairs* pairs, b2a_results* results, b2a_stats* stats);

/* banded::Aligner::{custom,global,semiglobal,local} (banded.rs:282,872,901,942)
 * with k-mer length k and band half-width w (banded.rs:150-180). */
int32_t b2a_align_batch_banded(b2a_engine* e, int32_t mode, const b2a_scoring* scoring,
                               uint32_t k, uint32_t w, const b2a_pairs* pairs,
                               b2a_results* results, b2a_stats* stats);

/* The banded::Aligner entry points that take the band's inputs from the caller (banded.rs:294-401, 938-975):
 *   custom_with_prehash / semiglobal_with_prehash   the k-mer hash of y only speeds the reference's match search
 *                                                   up; the matches, hence the results, are those of custom /
 *                                                   semiglobal: call b2a_align_batch_banded
 *   custom_with_matches(x, y, matches)              match_off + match_xy
 *   custom_with_expanded_matches(.., allowed_mismatches, use_lcskpp_union)
 *                                                   match_off + match_xy, allowed_mismatches (-1 = None),
 *                                                   use_lcskpp_union
 *   custom_with_match_path(x, y, matches, path)     match_off + match_xy + path_off + path_idx
 * Pair p's matches are (match_xy[2i], match_xy[2i+1]) = (xpos, ypos) for i in [match_off[p], match_off[p+1]),
 * its path the indices path_idx[path_off[p] .. path_off[p+1]) into those matches.  Where the reference panics
 * (matches not strictly ascending, a path index out of range, an empty path, positions outside the matrix) the
 * batch is refused with B2A_E_INVALID. */
typedef struct b2a_band_hints {
  const uint64_t* match_off; /* n_pairs + 1 */
  const uint32_t* match_xy;
  const uint64_t* path_off;  /* n_pairs + 1, or NULL */
  const uint32_t* path_idx;
  int32_t allowed_mismatches; /* -1: matches are used as given */
  int32_t use_lcskpp_union;
} b2a_band_hints;
int32_t b2a_align_batch_banded_hinted(b2a_engine* e, int32_t mode, const b2a_scoring* scoring,
                                      uint32_t k, uint32_t w, const b2a_pairs* pairs,
                                      const b2a_band_hints* hints, b2a_results* results, b2a_stats* stats);

/* banded::Aligner reduced to Alignment.score / xend / yend, as b2a_align_batch_scores is for Aligner: hints == NULL is
 * b2a_align_batch_banded, non-NULL hints are b2a_align_batch_banded_hinted (same validation and refusals).  For each
 * pair, score, xend and yend are what the full call returns.  The band (K4), the path every pair takes and the
 * per-pair statuses B2A_PAIR_CAPACITY / B2A_PAIR_INVALID_HINT are the full call's; a band above MAX_CELLS returns
 * MIN_SCORE, 0, 0 as there.  No interior traceback cell (1 <= i < m, 1 <= j < n) is stored, and the walk stops on the
 * first cell with i < m and j < n: xend and yend are set only by the suffix-clip moves, whose codes sit on row m and
 * column n, and the walk never increases i or j.  results: score, xend, yend and status; xstart, ystart, ops, ops_off
 * and clip_len must be NULL (else B2A_E_INVALID).  b2a_banded_band_ranges and b2a_banded_strip_pairs work after it
 * as after a full call.  status: a panic met on row m / column n is B2A_PAIR_PANIC; one only the interior walk would
 * meet (banded.rs:777-831) cannot be seen without the traceback, and such a pair reports its score. */
int32_t b2a_align_batch_banded_scores(b2a_engine* e, int32_t mode, const b2a_scoring* scoring, uint32_t k, uint32_t w,
                                      const b2a_pairs* pairs, const b2a_band_hints* hints, b2a_results* results,
                                      b2a_stats* stats);

/* Band::ranges of one pair of the last banded call (what banded::Aligner::visualize draws, banded.rs:1007-1030):
 * y_len + 1 half-open row ranges as (start, end) u32 pairs; an empty column is (x_len + 1, 0) (banded.rs:1065).
 * Kept on the device for the pairs of the call's last wave (every pair, unless the batch needed several waves). */
int32_t b2a_banded_band_ranges(b2a_engine* e, uint64_t pair, uint32_t* ranges, uint64_t capacity_pairs);

/* How many pairs of the last banded call K4 marked for the strip-wavefront fill (the packed-cell kernel for bands
 * whose starts and ends never decrease; the rest -- and the rare marked pair that path hands back -- ran the literal /
 * register-resident column loops of banded.rs:511-681).  A measurement aid: results do not depend on the path. */
int32_t b2a_banded_strip_pairs(b2a_engine* e, uint64_t* n_pairs);

/* Staged form of b2a_align_batch, so a caller can keep a batch resident in HBM:
 *   stage: validate, plan, host->device copy of the batch (async on the stream);
 *   run:   launch K0..K2 on the stream (async; may be called repeatedly);
 *   fetch: device->host copy of the results, stream-synchronised. */
int32_t b2a_batch_stage(b2a_engine* e, int32_t mode, const b2a_scoring* scoring,
                        const b2a_pairs* pairs);
int32_t b2a_batch_run(b2a_engine* e);
int32_t b2a_batch_fetch(b2a_engine* e, b2a_results* results, b2a_stats* stats);

/* Fixed-stride per-pair result records of the staged batch in DEVICE memory,
 * the unit that is all-gathered across GPUs (one ncclAllGather, SURVEY 8e):
 *   record = { int32 score; uint32 xstart, xend, ystart, yend, n_ops;
 *              uint32 clip_len[4]; uint8 ops[stride - 40] }.
 * Valid after b2a_batch_run until the next stage. */
int32_t b2a_batch_records(b2a_engine* e, void** dev_records, uint32_t* stride_bytes,
                          uint64_t* n_records);
/* Same records, but written into caller-provided DEVICE memory (e.g. a torch
 * tensor that is then handed to torch.distributed.all_gather_into_tensor). */
int32_t b2a_batch_records_into(b2a_engine* e, void* dev_dst, uint64_t dst_bytes,
                               uint32_t* stride_bytes);
uint32_t b2a_record_stride(uint32_t max_m, uint32_t max_n);

/* Decode host copies of gathered records into b2a_results (pure host code). */
int32_t b2a_records_decode(const void* host_records, uint32_t stride_bytes, uint64_t n_records,
                           b2a_results* results);

/* Compact form of the same results for the all-gather (what `bench.py --gpus N` and
 * rust_bio_b200/dist.py exchange): one segment per rank,
 *   { uint64 n_pairs; uint64 ops_bytes; uint8 pad[48]; }                       64 bytes
 *   int32 score[n]; uint32 xstart[n], xend[n], ystart[n], yend[n], n_ops[n]; uint32 clip_len[4n];
 *   uint8 ops[ops_bytes]                      (pair p's ops follow pair p-1's, b2a_results order)
 * i.e. 64 + 40 n + ops_bytes bytes instead of n * b2a_record_stride(): short alignments (local mode on
 * reads) travel at their real length.  b2a_batch_compact_bytes waits for the batch to finish and returns the
 * segment size; ranks agree on the largest one (a MAX all-reduce of one integer), each writes its segment
 * into a buffer of that size and a single all-gather moves them.
 * b2a_batch_compact_bytes / _into / _fixed also work after a full b2a_align_batch_banded / _hinted / _packed call:
 * its results stay on the device until the next call on the engine, and the segment is the same.  After a banded
 * call b2a_batch_run and b2a_batch_records* stay B2A_E_STATE (no batch is staged); after a score-only call (banded or
 * not) the compaction is B2A_E_STATE. */
int32_t b2a_batch_compact_bytes(b2a_engine* e, uint64_t* segment_bytes);
int32_t b2a_batch_compact_into(b2a_engine* e, void* dev_dst, uint64_t dst_bytes);
/* The same segment with a capacity the CALLER fixes (e.g. from the previous batch, or the bound
 * 64 + 40 n + sum(m + n + 4)): nothing here waits for the batch or reads a size back, so ranks need no size
 * agreement before the all-gather and the exchange of batch k can overlap the kernels of batch k + 1.  The header
 * is written on the device: { n_pairs, ops_bytes produced, ops_bytes kept (<= capacity), 0... }; a segment whose
 * ops did not fit is cut and says so (kept < produced) -- b2a_gathered_fetch refuses it (B2A_E_CAPACITY). */
int32_t b2a_batch_compact_fixed(b2a_engine* e, void* dev_dst, uint64_t capacity_bytes);
/* Reassembly on the rank that returns the results (SURVEY 8e: "rank 0's copy is what the shim returns"):
 * `dev_gathered` = n_segments segments of segment_bytes each, as all-gathered in DEVICE memory, in rank order.
 * Copies every field straight into `results` (host memory, pinned for speed) in that order and builds ops_off. */
int32_t b2a_gathered_fetch(b2a_engine* e, const void* dev_gathered, uint64_t segment_bytes, uint32_t n_segments,
                           b2a_results* results, uint64_t* n_pairs_total, uint64_t* d2h_bytes);
/* Decode one gathered segment (host memory) into `results` starting at pair index `pair_base` and ops offset
 * `ops_base`; returns the segment's pair count and ops bytes.  ops_off[pair_base + i] is written for every
 * pair of the segment (the caller writes the final ops_off[n_total]). */
int32_t b2a_compact_decode(const void* host_segment, uint64_t segment_bytes, uint64_t pair_base,
                           uint64_t ops_base, b2a_results* results, uint64_t* n_pairs, uint64_t* ops_bytes);

/* ---- every visible GPU from ONE process (SURVEY 8b / 8e; what a Rust caller of the shim uses on an 8-GPU node)
 * b2a_multi_create: one engine + one stream per device (device_ids == NULL / n_devices <= 0: all visible devices)
 * and an NCCL communicator over them (ncclCommInitAll, libnccl.so.2 bound at run time).
 * b2a_multi_align_batch: Aligner::{custom,global,semiglobal,local} over a batch with HOST inputs and outputs -- the
 * pair list is split contiguously into equal shares, every device stages and runs its share side by side, ONE
 * ncclAllGather of the compact result segments reassembles the per-pair results on every device, and device 0's copy
 * is decoded into `results`.  Bit-identical to b2a_align_batch on one device.  Without libnccl the segments are
 * gathered onto device 0 with peer copies instead; b2a_multi_exchange_kind() names what is in use.
 * A device list may name a device more than once: every entry gets its own engine and stream, no NCCL communicator is
 * made, and the segments are peer-copied onto entry 0.  The engines of one device size their scratch independently
 * (each from the free memory it sees: b2a_engine_set_traceback_budget), so shares that would fill a card on their own
 * can run it out of memory (B2A_E_CUDA) together; such a list is for testing and for measuring the split on one card.
 * A batch of fewer pairs than devices runs on device 0 alone.
 * results->status, when set, is filled per pair as on one engine (a failing pair marks only itself); without it such
 * a pair fails the call with the single engine's code and a "device N:" prefix on b2a_multi_last_error. */
typedef struct b2a_multi b2a_multi;
int32_t b2a_multi_create(b2a_multi** out, const int32_t* device_ids, int32_t n_devices);
int32_t b2a_multi_destroy(b2a_multi* m);
int32_t b2a_multi_device_count(const b2a_multi* m);
const char* b2a_multi_last_error(const b2a_multi* m);
const char* b2a_multi_exchange_kind(const b2a_multi* m);
int32_t b2a_multi_align_batch(b2a_multi* m, int32_t mode, const b2a_scoring* scoring, const b2a_pairs* pairs,
                              b2a_results* results, b2a_stats* stats);
/* banded::Aligner over every device: each device runs b2a_align_batch_banded (hints == NULL: the k-mer matches are
 * found on the device) or b2a_align_batch_banded_hinted on its share, then the shares are compacted, exchanged and
 * decoded as in b2a_multi_align_batch (same segments, one collective).  Bit-identical to the single-engine call; a band
 * above MAX_CELLS returns MIN_SCORE and no ops as there.  A hint list is checked over the whole batch before any device
 * runs (the single engine's rules, match_off and path_off ascending): a bad one is B2A_E_INVALID. */
int32_t b2a_multi_align_batch_banded(b2a_multi* m, int32_t mode, const b2a_scoring* scoring, uint32_t k, uint32_t w,
                                     const b2a_pairs* pairs, const b2a_band_hints* hints, b2a_results* results,
                                     b2a_stats* stats);
/* b2a_align_batch_scores and b2a_align_batch_banded_scores over every device, bit-identical to the single-engine
 * calls and under their output rules (score, xend, yend, status; the rest NULL).  Each device writes its share
 * straight into the caller's arrays: no ops, so no exchange. */
int32_t b2a_multi_align_batch_scores(b2a_multi* m, int32_t mode, const b2a_scoring* scoring, const b2a_pairs* pairs,
                                     b2a_results* results, b2a_stats* stats);
int32_t b2a_multi_align_batch_banded_scores(b2a_multi* m, int32_t mode, const b2a_scoring* scoring, uint32_t k,
                                            uint32_t w, const b2a_pairs* pairs, const b2a_band_hints* hints,
                                            b2a_results* results, b2a_stats* stats);
/* Stats of the b2a_multi_* calls: cells, h2d / d2h / traceback bytes and kernel launches are summed over the devices;
 * pack / band / fill / walk ms and waves are the slowest device's; the fill shape fields are device 0's. */

/* ---- bio::alignment::distance (reference src/alignment/distance.rs) over a batch of pairs: host arrays in, host arrays
 * out, single-shot.  Input checks are the aligner's (offsets inside seq_blob, at most 2^31 - 2 pairs); a sequence may be
 * up to 2^31 - 1 bytes.  distance[p] is pair p's result, in caller order.
 *   b2a_levenshtein_batch, k = B2A_DIST_NONE: levenshtein(x, y) == simd::levenshtein(x, y), the unit-cost edit distance
 *     over bytes.  Any other k: simd::bounded_levenshtein(x, y, k), i.e. the distance when it is <= min(k, max(|x|,
 *     |y|)), else B2A_DIST_NONE (None).  Myers/Hyyro bit-parallel columns, 64 rows per word; the engine picks, per pair,
 *     a thread with the pattern in registers (shorter side <= 256), a thread with a sliding band of words (bounded,
 *     k <= 223), or a warp (anything else).  Results do not depend on the choice.
 *   b2a_hamming_batch: hamming(x, y) == simd::hamming(x, y), the count of unequal positions.  A pair of unequal lengths
 *     (the reference panics) is B2A_PAIR_PANIC in `status` with distance B2A_DIST_NONE when status is set; without a
 *     status array it fails the call with B2A_E_INVALID.
 * stats: cells = sum of m * n (Levenshtein; for a bounded pair too, though the band computes fewer) or of m (Hamming),
 * pack_ms = the blob's rewrite into alphabet codes, fill_ms = the distance kernels, kernel_launches.
 * The multi forms split the pair list over the devices as b2a_multi_align_batch_scores does; each device writes its
 * share of distance (and status) straight into the caller's arrays.  Stats as for the other b2a_multi_* calls. */
#define B2A_DIST_NONE 0xFFFFFFFFu
int32_t b2a_levenshtein_batch(b2a_engine* e, uint32_t k, const b2a_pairs* pairs, uint32_t* distance, b2a_stats* stats);
int32_t b2a_hamming_batch(b2a_engine* e, const b2a_pairs* pairs, uint32_t* distance, uint32_t* status, b2a_stats* stats);
/* How many pairs of the last b2a_levenshtein_batch ran each way (a measurement aid; results do not depend on it):
 * counts[0] answered on the host (an empty side, or |m - n| above the bound), counts[1..4] a thread with the pattern's
 * 1..4 words in registers, counts[5] / counts[6] a thread with a 4- / 8-word band, counts[7] a warp.  Up to n_counts
 * (at most 8) entries are written. */
int32_t b2a_distance_tier_pairs(const b2a_engine* e, uint64_t* counts, uint32_t n_counts);
int32_t b2a_multi_levenshtein_batch(b2a_multi* m, uint32_t k, const b2a_pairs* pairs, uint32_t* distance,
                                    b2a_stats* stats);
int32_t b2a_multi_hamming_batch(b2a_multi* m, const b2a_pairs* pairs, uint32_t* distance, uint32_t* status,
                                b2a_stats* stats);

/* ---- bio::pattern_matching::myers (reference src/pattern_matching/myers) over a batch of (pattern x, text y) pairs.
 * The pattern is always x, also when it is longer than the text.  D[i][j] is the unit-cost edit distance with
 * D[0][j] = 0 (the text is free at both ends) and D[i][0] = i; pattern byte p matches text byte t when t == p, when
 * bit t of match->ambig row p is set (MyersBuilder::ambig: the pattern side only), or when t is a text wildcard
 * (MyersBuilder::text_wildcard).  match may be NULL, and either table in it.  Per pair:
 *   best_end[p], best_dist[p]: find_best_end, the FIRST end j - 1 (0-based) of the least D[m][j], and that distance
 *     (Myers::distance).  An empty text gives B2A_DIST_NONE for both.
 *   with n_hits set (a listing), every (j - 1, D[m][j]) with D[m][j] <= k, j = 1..n, in ascending end order
 *     (find_all_end); *n_hits = their total over the batch.  The hits stay on the engine until its next call of any
 *     kind and are copied out by b2a_myers_hits_fetch.  A listing whose hits (8 bytes each) are above the engine's
 *     device-memory budget (b2a_engine_set_traceback_budget; by default 60 % of the free memory) is refused with
 *     B2A_E_CAPACITY before the hits are allocated.  n_hits NULL: k is ignored and nothing is held.
 * An empty pattern (the reference panics: "Pattern is empty") is B2A_PAIR_PANIC in `status`, with best_end =
 * best_dist = B2A_DIST_NONE and no hits; without a status array it fails the call with B2A_E_INVALID naming the pair.
 * Myers/Hyyro bit-parallel columns over the batch's compacted alphabet: a thread with the pattern in registers up to
 * 256 symbols, a warp on 2048-row strips beyond.  Several pairs may share one x offset (one pattern, many texts).
 * stats: cells = sum of m * n, pack_ms = the blob's rewrite into alphabet codes, fill_ms = pass 1 (best ends and hit
 * counts), walk_ms = the listing's offsets and pass 2 (the pairs with hits rerun to write them), kernel_launches. */
typedef struct b2a_myers_match {
  const uint8_t* ambig;     /* NULL, or 256 rows x 32 bytes: bit t of row p = pattern byte p also matches text byte t */
  const uint8_t* wildcards; /* NULL, or 32 bytes: bit t = text byte t is matched by every pattern byte */
} b2a_myers_match;
int32_t b2a_myers_batch(b2a_engine* e, const b2a_myers_match* match, uint32_t k, const b2a_pairs* pairs,
                        uint32_t* best_end, uint32_t* best_dist, uint64_t* n_hits, uint32_t* status, b2a_stats* stats);
/* The held listing: hit_off[0..n_pairs] (pair p's hits are [hit_off[p], hit_off[p + 1])), hit_end and hit_dist of
 * *n_hits entries each.  B2A_E_STATE unless the engine's last call was b2a_myers_batch with a listing. */
int32_t b2a_myers_hits_fetch(b2a_engine* e, uint64_t* hit_off, uint32_t* hit_end, uint32_t* hit_dist);
/* How the pairs of the last b2a_myers_batch ran (a measurement aid; results do not depend on it): counts[0] answered
 * on the host (an empty side), counts[1..4] a thread with the pattern's 1..4 words in registers, counts[5] a warp,
 * counts[6] the pairs with hits that pass 2 reran.  Up to n_counts (at most 7) entries are written. */
int32_t b2a_myers_tier_pairs(const b2a_engine* e, uint64_t* counts, uint32_t n_counts);
/* The multi forms split the pair list as b2a_multi_levenshtein_batch does: each device writes its share of best_end,
 * best_dist (and status) at its offset, and *n_hits is the sum.  The fetch places each device's hits at its offset
 * with hit_off rebased; B2A_E_STATE unless the last b2a_multi_* call was b2a_multi_myers_batch with a listing. */
int32_t b2a_multi_myers_batch(b2a_multi* m, const b2a_myers_match* match, uint32_t k, const b2a_pairs* pairs,
                              uint32_t* best_end, uint32_t* best_dist, uint64_t* n_hits, uint32_t* status,
                              b2a_stats* stats);
int32_t b2a_multi_myers_hits_fetch(b2a_multi* m, uint64_t* hit_off, uint32_t* hit_end, uint32_t* hit_dist);

/* ---- bio::stats::pairhmm::PairHMM::prob_related (reference src/stats/pairhmm/pairhmm.rs) over a batch of (x, y) pairs:
 * the probability, summed over every alignment, that y is related to x, as a natural-log LogProb in f64.
 * prob[p] is pair p's result, in caller order, capped at 0 (ln_one) as the reference caps it.
 * Gap parameters are natural logs (GapParameters); free_start_gap_x / free_end_gap_x are StartEndGapParameters, with
 * prob_start_gap_x the trait's default.  max_edit_dist UINT64_MAX is None; any other value bands the recursion as the
 * reference does (Some(usize::MAX) gives the same results as None).
 * Emissions come in per-base classes: every sequence byte has a class byte at the same offset of class_blob (NULL:
 * every class is 0).  prob_emit_xy(i, j) = emit_match[cls(y[j])] when x[i] == y[j], else emit_mismatch[cls(y[j])];
 * prob_emit_x(i) = emit_x[cls(x[i])]; prob_emit_y(j) = emit_y[cls(y[j])].  A class byte >= n_classes is B2A_E_INVALID.
 * A gap parameter on which PairHMM::new's ln_one_minus_exp asserts (p <= 0.0) is B2A_E_INVALID.  A NaN result (the
 * reference's assert!(!p.is_nan())) is B2A_PAIR_PANIC in `status`, prob[p] NaN; without a status array it fails the
 * call with B2A_E_INVALID naming the pair.  Pairs with an empty side are answered on the host.
 * A warp per pair, lanes over y (strips of 256 columns beyond 256); several pairs may share one x offset (one window,
 * many reads).  stats: cells = sum of len_x * len_y (banded calls too: the band changes results, not the work),
 * fill_ms = the kernels, kernel_launches.
 * The multi form splits the pair list as b2a_multi_levenshtein_batch does; each device writes its share of prob (and
 * status) straight into the caller's arrays. */
typedef struct b2a_pairhmm_params {
  double prob_gap_x, prob_gap_y, prob_gap_x_extend, prob_gap_y_extend; /* GapParameters, natural log */
  int32_t free_start_gap_x, free_end_gap_x;                            /* StartEndGapParameters */
  uint64_t max_edit_dist;            /* UINT64_MAX = None */
  uint32_t n_classes;                /* 1 .. 256 */
  const double* emit_match;          /* [n_classes] each */
  const double* emit_mismatch;
  const double* emit_x;
  const double* emit_y;
  const uint8_t* class_blob;         /* NULL, or blob_bytes class bytes laid out like seq_blob */
} b2a_pairhmm_params;
int32_t b2a_pairhmm_batch(b2a_engine* e, const b2a_pairhmm_params* params, const b2a_pairs* pairs, double* prob,
                          uint32_t* status, b2a_stats* stats);
/* How the pairs of the last b2a_pairhmm_batch ran (a measurement aid; results do not depend on it): counts[0]
 * answered on the host (an empty side), counts[1..5] one strip with 1, 2, 4, 5, 8 columns per lane (len_y <= 32, 64,
 * 128, 160, 256), counts[6] strips of 256 columns.  Up to n_counts (at most 7) entries are written. */
int32_t b2a_pairhmm_tier_pairs(const b2a_engine* e, uint64_t* counts, uint32_t n_counts);
int32_t b2a_multi_pairhmm_batch(b2a_multi* m, const b2a_pairhmm_params* params, const b2a_pairs* pairs, double* prob,
                                uint32_t* status, b2a_stats* stats);

/* Measurement utility for the int32-ALU roofline (SURVEY 8d): tera lane-ops/s of
 * independent add / min-max / add+max register chains over all SMs of the device. */
int32_t b2a_util_int32_peak(int32_t device_id, float* tops_add, float* tops_minmax, float* tops_mixed);

#ifdef __cplusplus
}
#endif
#endif /* B200ALIGN_H_ */
