/*
 * bmb200.h -- C ABI of libbmb200: H100 (sm_90a) block-level set algebra for
 * BitMagic-format bit-vectors.
 *
 * This is the drop-in boundary for ONE path of tlk00/BitMagic: the 64 Kbit
 * block kernels behind bm::aggregator<>::combine_or / combine_and /
 * combine_and_sub, bm::bvector<>::bit_and/bit_or/bit_xor/bit_sub, bm::count_*
 * and the rank/select path (rs_index build, count_to, select).
 *
 * Conventions follow the reference's own C binding
 * (lang-maps/libbm/include/libbm.h:28-35,123-140): every function returns an
 * int error code (0 == OK), results come back through out-pointers, handles
 * are opaque, no C++ type or exception crosses the boundary.
 *
 * Reference interfaces replaced (file:line under the reference tree):
 *   bmb200_aggregate  OP_OR       <- aggregator::combine_or        src/bmaggregator.h:1101-1122,1626-1663
 *   bmb200_aggregate  OP_AND      <- aggregator::combine_and       src/bmaggregator.h:1126-1157,1668-1716
 *   bmb200_aggregate  OP_AND_SUB  <- aggregator::combine_and_sub   src/bmaggregator.h:1162-1220,1720-1803
 *   bmb200_aggregate  OP_XOR      <- bvector::bit_xor              src/bm.h:6072 (bit_block_xor src/bmfunc.h:9191)
 *   bmb200_aggregate  OP_SHIFT_R_AND <- aggregator::combine_shift_right_and  src/bmaggregator.h:2494-2669
 *   BMB200_F_COUNT_ONLY           <- bm::count_and/or/xor/sub      src/bmalgo.h:48-51, pipeline counts src/bmaggregator.h:1397
 *   bmb200_result_optimize        <- blocks_manager::opt_copy_bit_block src/bmblocks.h:1355-1409
 *   bmb200_set_upload_blobs       <- bm::deserialize / deserializer<BV>::deserialize  src/bmserial.h:4152,5578-6090
 *   bmb200_scan                   <- sparse_vector_scanner::find_eq/find_gt/find_ge/find_lt/find_le/find_range
 *                                                                   src/bmsparsevec_algo.h:1083-1182,2593-2632,4360-4395
 *   bmb200_rs_build               <- bvector::build_rs_index       src/bm.h:2531-2660, rs_index src/bmrs.h:688-715
 *   bmb200_rank_batch             <- bvector::count_to             src/bm.h:3120-3167
 *   bmb200_select_batch           <- bvector::select               src/bm.h:5350-5385
 *   bmb200_rank_decompress        <- rank_compressor::decompress   src/bmalgo.h:571-644,
 *                                    sparse_vector_scanner::decompress src/bmsparsevec_algo.h:4525-4537
 *   bmb200_rank_compress          <- rank_compressor::compress     src/bmalgo.h:498-566
 *
 * Block geometry (src/bmconst.h:55-68,78-87): a bit-block is 2048 x u32 =
 * 8192 B = 65536 bits; a GAP block is u16 buf[0..len], buf[0] = header
 * (bit0 = value of first run, bits1-2 = capacity level, bits3.. = len),
 * buf[1..len] = inclusive run-end positions, buf[len] == 65535.
 */
#ifndef BMB200_H_INCLUDED
#define BMB200_H_INCLUDED

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- error codes; 0..7 numerically identical to libbm.h:28-35 ---- */
#define BMB200_OK                  0
#define BMB200_ERR_BADALLOC        1
#define BMB200_ERR_BADARG          2
#define BMB200_ERR_RANGE           3
#define BMB200_ERR_RS_IDX_MISSING  7
#define BMB200_ERR_CUDA            200  /* a CUDA runtime call failed; see bmb200_last_error */
#define BMB200_ERR_NODEVICE        201  /* no sm_90 device: this library has NO CPU fallback */
#define BMB200_ERR_UNSUPPORTED     202  /* serialized BLOB uses a block encoding the device decoder does not cover */

/* ---- geometry ---- */
#define BMB200_BLOCK_WORDS     2048u
#define BMB200_BLOCK_BYTES     8192u
#define BMB200_BLOCK_BITS      65536u
#define BMB200_GAP_MAX_WORDS   1280u     /* src/bmconst.h:80  gap_max_buff_len */
#define BMB200_GAP_THRESHOLD   1276u     /* glen(max_level)-4, src/bmblocks.h:1391 */
#define BMB200_GAP_UNIT_WORDS  8u        /* GAP blocks start on 16-byte units in the arena */
#define BMB200_SUPERBLOCK      256u      /* blocks per top-level entry, src/bmconst.h:95 */

/* block kinds (2 bits); mirror the four pointer states of src/bmdef.h:165-199 */
#define BMB200_BLK_NULL  0u
#define BMB200_BLK_FULL  1u
#define BMB200_BLK_BIT   2u
#define BMB200_BLK_GAP   3u
#define BMB200_DESC_GAP_PAD  0x80000000u   /* GAP block stored with a 2-byte lead pad (see bmb200_packed_set) */
#define BMB200_DESC_GAP_FLAT 0x40000000u   /* GAP block stored in the flat-streamable form (see bmb200_packed_set) */
#define BMB200_DESC_REL_MASK 0x0fffffffu   /* rel = (desc >> 2) & mask */

/* ---- operations ---- */
#define BMB200_OP_OR       0   /* group0 = sources                       */
#define BMB200_OP_AND      1   /* group0 = sources                       */
#define BMB200_OP_AND_SUB  2   /* group0 = AND sources, group1 = SUB set */
#define BMB200_OP_XOR      3   /* group0 = sources (2-operand in the reference, N-way here) */
#define BMB200_OP_SHIFT_R_AND 4 /* group0 = v_0 .. v_{n-1} IN ORDER: T_0 = v_0, T_k = (T_{k-1} >> 1) & v_k, result = T_{n-1}
                                 * (aggregator::combine_shift_right_and; ">> 1" = every bit to the next higher index);
                                 * n <= 65536.  Bits pushed past the last block column of the set are dropped: give the
                                 * set one spare (NULL) column if the sources can carry out of their last block. */

#define BMB200_OP_SUB      5   /* bmb200_binop only: a AND NOT b (bvector::bit_sub) */

/* ---- flags for bmb200_aggregate ---- */
#define BMB200_F_COUNT_ONLY  1u  /* per-column popcount/digest only; no result blocks stored */
#define BMB200_F_OPT_NONE    0u  /* result kinds as aggregator opt_mode_ == opt_none           */
#define BMB200_F_OPT_COMPRESS 2u /* classify + bit->GAP like opt_copy_bit_block(opt_compress) */
#define BMB200_F_OR_TARGET   4u  /* batch only: also accumulate the union of all group results (pipeline::set_or_target) */

typedef struct bmb200_ctx    bmb200_ctx;     /* one per process per GPU                      */
typedef struct bmb200_set    bmb200_set;     /* device-resident column-major set of vectors  */
typedef struct bmb200_result bmb200_result;  /* device-resident aggregate result             */
typedef struct bmb200_rs     bmb200_rs;      /* device-resident rank-select index            */

/*
 * Packed (column-major) set of n_vec vectors x n_blocks block columns.
 *   desc[nb*n_vec + v] = kind | (rel << 2)
 *      BIT: rel = index of the block inside column nb's bit segment
 *      GAP: rel = offset inside column nb's GAP segment, in 16-byte units (28 bits).
 *           bit 31 (BMB200_DESC_GAP_PAD): the block is stored after ONE leading u16 of padding.
 *           bit 30 (BMB200_DESC_GAP_FLAT): the block is in the flat-streamable form --
 *             - the (previous run end, run end) u16 pair of every 1-run is a 4-byte aligned word: a block whose
 *               first run is 0 carries the lead pad, a block whose first run is 1 does not;
 *             - the lead pad holds 0xFFFF and the bytes between buf[len] and the next 16-byte unit hold 0, so
 *               header, pad, terminator and fill all read as pairs with first >= second (= no run);
 *             - the units between two FLAT blocks of a column hold nothing else (no holes with stale data).
 *           A window of FLAT blocks is then a plain array of 1-runs that the aggregation kernel consumes with
 *           128-bit shared loads and no per-block work (agg_kernel.cuh).  Both bits are optional per block:
 *           every kernel accepts every form; the library's own packers and bmb200_synth_set write FLAT.
 *   bit segment of column nb = bit_pool blocks [bit_base[nb], bit_base[nb+1])
 *   GAP segment of column nb = gap_pool units  [gap_base[nb], gap_base[nb+1])
 *   Every block of a segment belongs to exactly one vector of its column (no unreferenced or shared blocks): an aggregation
 *   over the whole set reads the segments as they lie.
 * All blocks of one column are contiguous, so one CTA streams one column.
 */
typedef struct bmb200_packed_set {
    uint32_t        n_vec;
    uint32_t        n_blocks;
    const uint32_t* desc;      /* [n_blocks * n_vec]            */
    const uint64_t* bit_base;  /* [n_blocks + 1], in blocks     */
    const uint64_t* gap_base;  /* [n_blocks + 1], in 16-B units */
    const uint32_t* bit_pool;  /* bit_base[n_blocks] * 2048 u32 */
    const uint16_t* gap_pool;  /* gap_base[n_blocks] * 8 u16    */
} bmb200_packed_set;

/* One vector as the host block tree sees it: kind + pointer per block slot
 * (what blocks_manager::get_block_ptr(i,j) yields, src/bmblocks.h:556). */
typedef struct bmb200_vec_blocks {
    uint32_t           n_blocks;
    const uint8_t*     kind;   /* [n_blocks] BMB200_BLK_*                        */
    const void* const* ptr;    /* [n_blocks] 8 KB bit-block or GAP buf, else 0   */
} bmb200_vec_blocks;

typedef struct bmb200_agg_args {
    int32_t         op;        /* BMB200_OP_*                                    */
    uint32_t        flags;     /* BMB200_F_*                                     */
    const uint32_t* group0;    /* vector indices inside the set                  */
    uint32_t        n0;
    const uint32_t* group1;    /* SUB group for OP_AND_SUB, else ignored         */
    uint32_t        n1;
    uint32_t        nb_from;   /* block-column range [nb_from, nb_to)            */
    uint32_t        nb_to;     /* 0 == n_blocks                                  */
} bmb200_agg_args;

/* A pipeline batch: n_groups argument groups over ONE shared set (aggregator::pipeline, src/bmaggregator.h:222-341).
 * Group g uses members[offsets[2g] .. offsets[2g+1]) as group0 (AND / OR / XOR sources) and
 * members[offsets[2g+1] .. offsets[2g+2]) as group1 (SUB sources, OP_AND_SUB only). */
typedef struct bmb200_batch_args {
    int32_t         op;
    uint32_t        flags;      /* BMB200_F_* ; BMB200_F_COUNT_ONLY = pipeline<agg_opt_only_counts> */
    uint32_t        n_groups;
    const uint32_t* members;    /* vector indices inside the set, all groups concatenated */
    const uint32_t* offsets;    /* [2 * n_groups + 1] */
    uint32_t        nb_from;
    uint32_t        nb_to;      /* 0 == n_blocks */
} bmb200_batch_args;

/* Per-column result metadata (host arrays of n_cols = nb_to - nb_from entries; any may be NULL) */
typedef struct bmb200_result_meta {
    uint8_t*  kind;     /* BMB200_BLK_* after the opt-mode classification         */
    uint32_t* popcnt;   /* bits set in the column's result block                  */
    uint64_t* digest;   /* 64-wave non-zero bitmap, calc_block_digest0 src/bmfunc.h:1239 */
    uint32_t* nruns;    /* bit_block_calc_change of the result, src/bmfunc.h:6040  */
} bmb200_result_meta;

/* ---------------- context ---------------- */
int bmb200_init(int device, bmb200_ctx** out);
int bmb200_destroy(bmb200_ctx* ctx);
const char* bmb200_error_msg(int code);
/* text of the last CUDA failure seen by this context (empty string if none) */
int bmb200_last_error(const bmb200_ctx* ctx, char* buf, size_t buflen);
/* run all work of this context on an existing cudaStream_t (e.g. torch's current stream) */
int bmb200_ctx_set_stream(bmb200_ctx* ctx, void* cuda_stream);
int bmb200_ctx_get_stream(const bmb200_ctx* ctx, void** cuda_stream);
int bmb200_ctx_sync(bmb200_ctx* ctx);
/* number of kernels this context has launched so far */
int bmb200_ctx_launch_count(const bmb200_ctx* ctx, uint64_t* out);
int bmb200_device_info(const bmb200_ctx* ctx, int* sm_count, int* cc_major, int* cc_minor, uint64_t* hbm_bytes);
/* tuning knobs (results never depend on them): key 0 = GAP phase mode (0 auto: stream sorted member lists
 * through the shared-memory ring, 1 always gather), key 1 = resident CTAs per SM of the aggregation kernel */
#define BMB200_TUNE_GAP_MODE     0
#define BMB200_TUNE_CTAS_PER_SM  1
#define BMB200_TUNE_HOST_THREADS 2   /* host threads that pack blocks in bmb200_set_upload_vectors: 0 = all cores (at most 64) */
#define BMB200_TUNE_AGG_PIPELINE 3   /* 1 (default) = whole-set AND-SUB aggregations take the streamed-column kernel, 0 = never (A/B reference) */
#define BMB200_TUNE_RUN_LISTS    4   /* run-list companion of a set's GAP blocks, streamed by the whole-set AND-SUB kernel when the AND group
                                        holds no GAP block: 1 (default) = built on the set's second such call, 2 = on its first, 0 = never */
int bmb200_ctx_set_tuning(bmb200_ctx* ctx, int key, int value);
/* pin the CALLING thread (and the threads it starts later, e.g. the packers of bmb200_set_upload_vectors) to the CPUs of the NUMA
 * node this context's GPU hangs off, so that pinned staging memory is allocated next to the GPU's PCIe root.  *node = the node, or
 * -1 when the box has no NUMA information (then nothing is changed).  Call it before the first upload. */
int bmb200_ctx_bind_host_numa(bmb200_ctx* ctx, int* node);
/* bmb200_set_free parks the device arena of the set it frees in the context (at most one) and the next upload that fits reuses it,
 * so per-call uploads do not pay cudaMalloc / cudaFree of a multi-GB arena every time; bmb200_set_upload_slabs likewise keeps its
 * device mirror of the host slabs for the next call.  bmb200_ctx_trim gives all of that memory back */
int bmb200_ctx_trim(bmb200_ctx* ctx);

/* ---------------- sets ---------------- */
/* copy a packed set from HOST memory (pinned or pageable) into HBM */
int bmb200_set_upload(bmb200_ctx* ctx, const bmb200_packed_set* host, bmb200_set** out);
/* gather per-vector block pointers (the host block tree) into a packed device set.  The blocks are packed by a team of host
 * threads (BMB200_TUNE_HOST_THREADS) into a ring of pinned staging slots owned by the context and copied chunk by chunk, packing
 * and DMA overlapped; the set then stays resident until bmb200_set_free (bm::b200::device_set in the C++ binding).
 * To upload only a shard, pass kind + nb_from / ptr + nb_from with n_blocks = the shard's width. */
int bmb200_set_upload_vectors(bmb200_ctx* ctx, uint32_t n_vec, uint32_t n_blocks,
                              const bmb200_vec_blocks* vecs, bmb200_set** out);
/* The same upload for vectors whose blocks live inside a few large HOST SLABS (a slab-backed block allocator in the place of
 * bm::block_allocator, src/bmalloc.h:57-98 -- the seam sample6.cpp:47-110 shows -- or the arenas of frozen vectors,
 * src/bmblocks.h:2607-2771): no host thread touches a block.  The slabs cross PCIe as they lie (one DMA each, at link speed when
 * they are pinned: bmb200_host_slab_alloc), the block tree is walked and laid out WHILE they are in flight, and one kernel then
 * gathers the blocks from the device mirror into the column-major arena (same arena, descriptors and results as
 * bmb200_set_upload_vectors).  Every BIT / GAP block pointer must lie inside one of the slabs and be 32-byte aligned, and
 * the slabs may hold up to 128 GB together; when that does not hold the call falls back to bmb200_set_upload_vectors. */
typedef struct bmb200_host_slab {
    const void* base;    /* start of the slab                                                            */
    uint64_t    bytes;   /* bytes in use from base (the extent that is copied)                           */
} bmb200_host_slab;
int bmb200_set_upload_slabs(bmb200_ctx* ctx, uint32_t n_vec, uint32_t n_blocks, const bmb200_vec_blocks* vecs,
                            const bmb200_host_slab* slabs, uint32_t n_slabs, bmb200_set** out);
/* optional: queue the DMA of the slabs BEFORE the caller walks its block trees (the walk then runs under the copies too); the next
 * bmb200_set_upload_slabs on this context with the same slab list picks the copies up instead of issuing them again */
int bmb200_host_slabs_prefetch(bmb200_ctx* ctx, const bmb200_host_slab* slabs, uint32_t n_slabs);
/* page-locked host memory for such slabs (cudaHostAlloc, portable across the GPUs of the process).  No context needed. */
int bmb200_host_slab_alloc(uint64_t bytes, void** out);
int bmb200_host_slab_free(void* slab);
/* deserialize-to-device: vector v of the set arrives as a BitMagic serialization BLOB (bm::serializer<>, src/bmserial.h) and
 * is decoded on the GPU straight into the arena -- what bm::deserialize(bv, buf) (src/bmserial.h:4152) + an upload of the
 * materialised blocks would produce (same bits, same block kinds), with only the compressed bytes crossing PCIe.
 * Covered: every block encoding bm::serializer<> of this reference version writes for a plain bvector at compression levels
 * 0..6 (6 = its default): the explicit-length ones (zero / one runs, plain bit, bit interval, bit 0-runs, bit digest0, single
 * bit, bit / GAP position arrays, GAP with 16-bit run ends) are located by a host walk of the token bytes and decoded one CTA
 * per block; as soon as one BLOB of the call holds an entropy-coded token (Elias-gamma arrays and GAP blocks, binary
 * interpolative GAP / bit-array blocks v3 / v3s with delta-range reduction and exception lists, super-block position lists,
 * bookmarks) the token streams are walked ON THE DEVICE (one warp per vector, csrc/blob_entropy.cuh) and every entropy-coded
 * token is then decoded by a warp of its own.  Not covered (BMB200_ERR_UNSUPPORTED, no CPU fallback): XOR-reference compression
 * (BM_HM_HXOR, sparse-vector serialization), id-list streams, and the legacy encodings the reference can
 * still read but no longer writes (tokens 20, 27-29, 31, 32, 43-45, 56, 57).  Malformed / truncated streams: BMB200_ERR_BADARG. */
typedef struct bmb200_blob { const void* data; uint64_t size; } bmb200_blob;
int bmb200_set_upload_blobs(bmb200_ctx* ctx, uint32_t n_vec, uint32_t n_blocks, const bmb200_blob* blobs, bmb200_set** out);
/* adopt pointers that already live in HBM (caller keeps ownership of the memory) */
int bmb200_set_adopt_device(bmb200_ctx* ctx, const bmb200_packed_set* dev, bmb200_set** out);
/* sizes: total bit blocks, total GAP 16-B units, stored bytes of all source blocks */
int bmb200_set_info(const bmb200_set* set, uint32_t* n_vec, uint32_t* n_blocks,
                    uint64_t* n_bit_blocks, uint64_t* n_gap_units);
/* copy columns [nb_from, nb_to) back to caller-provided host buffers.
 * desc: (nb_to-nb_from)*n_vec u32; bit_base/gap_base: (nb_to-nb_from+1) u64, rebased to 0;
 * bit_pool / gap_pool sized from bmb200_set_column_sizes. */
int bmb200_set_column_sizes(const bmb200_set* set, uint32_t nb_from, uint32_t nb_to,
                            uint64_t* n_bit_blocks, uint64_t* n_gap_units);
int bmb200_set_download(const bmb200_set* set, uint32_t nb_from, uint32_t nb_to,
                        uint32_t* desc, uint64_t* bit_base, uint64_t* gap_base,
                        uint32_t* bit_pool, uint16_t* gap_pool);
/* device addresses of the packed arrays (for torch / NCCL interop) */
int bmb200_set_device_ptrs(const bmb200_set* set, bmb200_packed_set* out);
int bmb200_set_free(bmb200_set* set);
/* bytes of the set's run-list companion (BMB200_TUNE_RUN_LISTS): singles part and long-run part; 0 / 0 while none is built.
 * It is freed with the set. */
int bmb200_set_run_lists(const bmb200_set* set, uint64_t* sgl_bytes, uint64_t* lr_bytes);
/* part B of the companion: the listed runs of the set's sparse bit-blocks (singles and long-run bytes) and how many bit-blocks it
 * lists; 0 / 0 / 0 while none is built.  bmb200_set_run_lists reports part A, the runs of the GAP blocks. */
int bmb200_set_bit_run_lists(const bmb200_set* set, uint64_t* sgl_bytes, uint64_t* lr_bytes, uint64_t* listed_blocks);

/* synthetic input generator (bench / test support): vector v has iid bit density
 * density[v], counter-based RNG keyed by seed[v]; with optimize != 0 every block is
 * stored the way bvector::optimize(opt_compress) would store it (NULL/FULL/GAP/BIT). */
int bmb200_synth_set(bmb200_ctx* ctx, uint32_t n_vec, uint32_t n_blocks,
                     const double* density, const uint64_t* seed, int optimize,
                     bmb200_set** out);

/* ---------------- aggregation ---------------- */
/* asynchronous on the context stream; result stays in HBM until fetched or freed.
 * *reuse (may be NULL): pass a previous result of the same shape to recycle its buffers. */
int bmb200_aggregate(bmb200_ctx* ctx, const bmb200_set* set, const bmb200_agg_args* args,
                     bmb200_result** inout);
/* Two-operand bvector ops with the reference's result KINDS: target = a OP b for bvector::bit_or / bit_and / bit_xor / bit_sub
 * (src/bm.h:5973,6185,6072,6403; op = BMB200_OP_OR / _AND / _XOR / _SUB).  Per block column the kind of the result follows
 * combine_operation_block_or/_and/_xor/_sub (src/bm.h:6945,7100,7018,7285): a NULL / FULL argument clones the other block in
 * its own kind, GAP x GAP is MERGED as run lists on the device (gap_buff_op, src/bmfunc.h:3747: no 8 KB expansion; result GAP,
 * all-zero -> nothing, too long -> bit-block), GAP x bit and bit x bit give a bit-block that only BMB200_F_OPT_COMPRESS
 * re-classifies (optimize_bit_block).  calc_stat() of the stored result equals the reference's.  flags: F_OPT_NONE / F_OPT_COMPRESS. */
int bmb200_binop(bmb200_ctx* ctx, const bmb200_set* set, int op, uint32_t va, uint32_t vb, uint32_t flags,
                 uint32_t nb_from, uint32_t nb_to, bmb200_result** inout);
/* aggregator::combine_and_sub(TPipe&) (src/bmaggregator.h:1291-1453): every group in ONE launch.  The result has
 * n_groups * n_cols columns, group-major (column c of group g at index g * n_cols + c); metadata / fetch calls work
 * on that flat range. */
int bmb200_aggregate_batch(bmb200_ctx* ctx, const bmb200_set* set, const bmb200_batch_args* args, bmb200_result** inout);
/* per-group cardinalities (pipeline::get_bv_count_vector) */
int bmb200_result_group_totals(bmb200_result* res, uint64_t* totals, uint32_t n_groups);
/* finalize the OR target of a batch launched with BMB200_F_OR_TARGET into its own n_cols-column result */
int bmb200_result_or_target(bmb200_result* res, bmb200_result** out);
/* classify every result column like opt_copy_bit_block and convert runs < 1276 to GAP on device */
int bmb200_result_optimize(bmb200_result* res);
/* total popcount over all columns and "any bit found" (combine_and_sub's return value) */
int bmb200_result_total(bmb200_result* res, uint64_t* total, int* any);
int bmb200_result_fetch_meta(bmb200_result* res, const bmb200_result_meta* out);
/* ONE column of a result: *kind = BMB200_BLK_*; a BIT column fills bits[2048], a GAP column fills gaps[BMB200_GAP_MAX_WORDS]
 * (header + run ends), NULL / FULL columns write nothing.  What aggregator::find_first_and_sub reads after it has located the
 * first non-empty column from the popcounts (bm::bit_find_first on the temp block, src/bmaggregator.h:1538-1546). */
int bmb200_result_fetch_column(bmb200_result* res, uint32_t col, uint8_t* kind, uint32_t* bits, uint16_t* gaps);
/* sizes of the compacted result: BIT blocks and GAP u16 words (each GAP block padded to 8 words) */
int bmb200_result_sizes(bmb200_result* res, uint64_t* n_bit_blocks, uint64_t* n_gap_words);
/* compacted result in per-vector flat form: off[c] = index into bits (blocks) for BIT columns,
 * offset into gaps (u16 words) for GAP columns */
int bmb200_result_fetch(bmb200_result* res, uint8_t* kind, uint64_t* off,
                        uint32_t* bits, uint16_t* gaps);
/* same result, delivered into pinned host memory OWNED BY THE CONTEXT (no allocation once warm, two stream synchronisations):
 * kind[n_cols], off[n_cols], bits, gaps as in bmb200_result_fetch; *total = cardinality over all groups.  The pointers stay
 * valid until the next bmb200_result_fetch_view on the same context.  This is the call a resident-set ("warm") aggregation
 * ends with: bm::b200::aggregator materialises its target bvector from these views. */
int bmb200_result_fetch_view(bmb200_result* res, const uint8_t** kind, const uint64_t** off, const uint32_t** bits,
                             const uint16_t** gaps, uint64_t* n_bit_blocks, uint64_t* n_gap_words, uint64_t* total);
/* the same views, handed out as soon as kind[] / off[] are known: the blocks are still arriving, in column order, in up to 8
 * chunks.  bmb200_result_fetch_wait(res, col) returns once every block of the columns [0, col] has landed (callable from several
 * threads); the caller then reads bits / gaps of those columns.  bm::b200::aggregator stores the first columns into the target
 * bvector while the last ones are still crossing PCIe.  Wait for the last column before the next fetch on this context. */
int bmb200_result_fetch_view_async(bmb200_result* res, const uint8_t** kind, const uint64_t** off, const uint32_t** bits,
                                   const uint16_t** gaps, uint64_t* n_bit_blocks, uint64_t* n_gap_words, uint64_t* total);
int bmb200_result_fetch_wait(bmb200_result* res, uint32_t col);
/* device addresses: blocks [n_cols][2048] u32, popcnt [n_cols] u32, digest [n_cols] u64, flag [n_cols] u8 */
int bmb200_result_device_ptrs(const bmb200_result* res, void** blocks, void** popcnt,
                              void** digest, void** flag, uint32_t* n_cols);
int bmb200_result_free(bmb200_result* res);

/* ---------------- sparse-vector scanner (bit-sliced comparison) ---------------- */
/* sparse_vector_scanner<SV> searches over the bit-planes ("slices", bm::sparse_vector::get_slice(i),
 * src/bmsparsevec.h) of ONE unsigned sparse vector stored as vectors of a set: plane j (bit j of every element) is set
 * vector plane0 + j.  One launch answers n_values searches; the result has n_values * n_cols columns, value-major,
 * exactly like a pipeline batch (per-value cardinalities through bmb200_result_group_totals). */
#define BMB200_SCAN_EQ     0   /* find_eq    src/bmsparsevec_algo.h:1083  elements == value                    */
#define BMB200_SCAN_GT     1   /* find_gt    :1135                        elements >  value                    */
#define BMB200_SCAN_GE     2   /* find_ge    :1144                                                             */
#define BMB200_SCAN_LT     3   /* find_lt    :1154                                                             */
#define BMB200_SCAN_LE     4   /* find_le    :1163                                                             */
#define BMB200_SCAN_RANGE  5   /* find_range :1174  values[2k] <= element <= values[2k+1] (reversed bounds are swapped, :2871) */
typedef struct bmb200_scan_args {
    uint32_t        plane0;     /* first plane vector inside the set                                          */
    uint32_t        n_planes;   /* 1..64 (sparse_vector::effective_slices())                                  */
    uint32_t        universe;   /* set vector with the searchable indexes: [0, size) for a non-nullable vector,
                                 * the NOT-NULL plane for a nullable one (what finalize_search_result and
                                 * invert_internal apply, :2426,1686); 0xffffffff = every index of the columns */
    int32_t         pred;       /* BMB200_SCAN_*                                                              */
    uint32_t        flags;      /* BMB200_F_COUNT_ONLY / BMB200_F_OPT_COMPRESS                                */
    const uint64_t* values;     /* HOST: n_values search values (RANGE: 2 * n_values, lo then hi)             */
    uint32_t        n_values;
    uint32_t        nb_from;
    uint32_t        nb_to;      /* 0 == n_blocks */
} bmb200_scan_args;
int bmb200_scan(bmb200_ctx* ctx, const bmb200_set* set, const bmb200_scan_args* args, bmb200_result** inout);

/* end-to-end convenience: HOST packed set in, HOST metadata out, in one call: H2D of the whole set (every call), kernel,
 * D2H of the per-column metadata requested in meta_out (kind / popcnt / digest / nruns) and of the cardinality.  The result
 * blocks stay on the device (fetch them with bmb200_result_fetch on a result of bmb200_aggregate when they are needed). */
int bmb200_aggregate_host(bmb200_ctx* ctx, const bmb200_packed_set* host,
                          const bmb200_agg_args* args, const bmb200_result_meta* meta_out,
                          uint64_t* total_out);

/* ---------------- multi-GPU: block-range shards + ONE exchange (one process per GPU) ----------------
 * Every block column is independent (the reference loops (i,j) without carried state, src/bmaggregator.h:1113-1121,1184-1218),
 * so rank g of G owns a contiguous, superblock-aligned range of block columns of EVERY vector, uploads and aggregates only that
 * range, and the ranks exchange the per-column popcounts (4 B / column) and their cardinalities with one ncclAllGather over
 * NVLink / NVSwitch.  NCCL is bound at run time (dlopen libnccl.so.2); BMB200_ERR_UNSUPPORTED when it cannot be found. */
#define BMB200_COMM_ID_BYTES 128                       /* = sizeof(ncclUniqueId) */
int bmb200_shard_range(uint32_t n_blocks, int nranks, int rank, uint32_t* nb_from, uint32_t* nb_to);
/* rank 0: create the id and hand the 128 bytes to the other ranks (MPI / sockets / torch.distributed ...) */
int bmb200_comm_unique_id(void* id);
/* collective over all ranks: one communicator + one side stream per context */
int bmb200_comm_init(bmb200_ctx* ctx, int nranks, int rank, const void* id);
int bmb200_comm_info(const bmb200_ctx* ctx, int* nranks, int* rank);
int bmb200_comm_destroy(bmb200_ctx* ctx);
/* exchange of the local result `res` (single group) with all ranks; asynchronous, ordered after the work already queued on the
 * context stream; buffered three deep (the aggregation of step i never waits for the exchange of step i-1 or i-2).  Collective: every rank issues the same
 * sequence of exchanges.  Two transports (bmb200_exchange_mode):
 *   1 = one ncclAllGather of the rows on the context's SIDE stream (the default: the faster of the two where it was measured);
 *   2 = peer memory (BMB200_EXCHANGE_DIRECT=1): every rank's exchange buffer is mapped by every other rank through CUDA IPC and
 *       a small kernel behind the aggregation kernel stores this rank's (popcounts | cardinality) row into all of them over
 *       NVLink and publishes a sequence number; falls back to 1 when a rank cannot map a peer.
 * cols_per_rank = the width of the widest shard (the same value on every rank; narrower shards are zero-padded), 0 = the
 * result's own column count when all shards are equal. */
int bmb200_exchange_popcounts(bmb200_result* res, uint32_t cols_per_rank);
/* *mode = 0 before the first exchange (or without a communicator), else the transport in use (see above) */
int bmb200_exchange_mode(const bmb200_ctx* ctx, int* mode);
/* make the context stream wait for every exchange issued so far (asynchronous) */
int bmb200_exchange_fence(bmb200_ctx* ctx);
/* wait for the LAST exchange and read it: global cardinality, per-rank cardinalities [nranks], per-column popcounts of every
 * shard [nranks * n_cols] (host; any may be NULL); *d_gathered = the same data in HBM, rank r's columns at r * *stride u32 */
int bmb200_exchange_fetch(bmb200_ctx* ctx, uint64_t* global_total, uint64_t* rank_totals, uint32_t* popcnt,
                          const uint32_t** d_gathered, uint32_t* stride);

/* ---------------- rank / select ---------------- */
/* build the rs_index of vector `vec` of `set`; the set must outlive the index */
int bmb200_rs_build(bmb200_ctx* ctx, const bmb200_set* set, uint32_t vec, bmb200_rs** out);
/* recompute the index in place (same set, same vector) -- e.g. after the arena was refilled; no allocation */
int bmb200_rs_rebuild(bmb200_rs* rs);
/* index fields exactly as rs_index::register_super_block receives them (src/bmrs.h:688):
 * bcount[n_blocks] u32, sub_count[n_blocks] u64 (first | second<<16 | aux0<<32 | aux1<<48),
 * sb_count[n_superblocks+1] u64 running totals (sblock_count_) */
int bmb200_rs_export(bmb200_rs* rs, uint32_t* bcount, uint64_t* sub_count, uint64_t* sb_count);
int bmb200_rs_total(bmb200_rs* rs, uint64_t* total_bits_set);
/* inclusive rank: out[q] = number of set bits in [0, pos[q]]   (bvector::count_to) */
int bmb200_rank_batch(bmb200_rs* rs, const uint64_t* pos, uint64_t n, uint64_t* out);
/* 1-based select: found[q] = 0 for rank 0 or rank > count      (bvector::select)   */
int bmb200_select_batch(bmb200_rs* rs, const uint64_t* rank, uint64_t n, uint64_t* pos, uint8_t* found);
/* same, queries and answers already in HBM (asynchronous on the context stream) */
int bmb200_rank_batch_dev(bmb200_rs* rs, const uint64_t* d_pos, uint64_t n, uint64_t* d_out);
int bmb200_select_batch_dev(bmb200_rs* rs, const uint64_t* d_rank, uint64_t n, uint64_t* d_pos, uint8_t* d_found);
int bmb200_rs_free(bmb200_rs* rs);

/* ---------------- rank compression (rank-select compressed sparse vectors) ----------------
 * A bm::rsc_sparse_vector<> (src/bmsparsevec_compr.h) keeps only its NOT-NULL elements in its bit-planes, packed to the
 * positions [0, effective_size()); its NOT-NULL vector NN maps them back to the logical index space.  A search over it is a
 * bmb200_scan over the compressed columns [0, ceil(effective_size / 65536)) with the universe [0, effective_size), followed
 * by bmb200_rank_decompress with the rs index of NN (sparse_vector_scanner searches an RSC vector the same way,
 * src/bmsparsevec_algo.h:2300-2306,4525-4537).  A count-only search needs no decompression: it is a bijection on the bits
 * below count(NN), so the scan's group totals are already the answer.  flags: BMB200_F_OPT_NONE / BMB200_F_OPT_COMPRESS. */
/* rank_compressor<BV>::decompress  src/bmalgo.h:571 ; sparse_vector_scanner::decompress src/bmsparsevec_algo.h:4525
 * idx = the rs index of the NOT-NULL vector (bmb200_rs_build); src = any result whose columns start at compressed column 0
 * (n_groups groups of cols_per_group columns).  Out: n_groups * n_blocks(idx) columns, group-major, like a pipeline batch.
 * Bit p of group g is set iff NN[p] is set and bit rank_NN(p) - 1 of group g of src is set; compressed positions past the
 * source's columns read as 0, positions >= count(NN) are never read. */
int bmb200_rank_decompress(bmb200_ctx* ctx, const bmb200_rs* idx, const bmb200_result* src, uint32_t flags, bmb200_result** inout);
/* rank_compressor<BV>::compress  src/bmalgo.h:498 ; src = vector src_vec of the set idx was built on; bits outside idx dropped.
 * Out: one group of max(1, ceil(count(idx) / 65536)) columns.  Bit r is set iff src is set at the position of the (r+1)-th set
 * bit of NN.  For src not a subset of NN the result is compress(src & NN); the reference requires src to be a subset
 * (src/bmalgo.h:526-549, asserted only) and computes an unspecified result otherwise. */
int bmb200_rank_compress(bmb200_ctx* ctx, const bmb200_rs* idx, uint32_t src_vec, uint32_t flags, bmb200_result** inout);

#ifdef __cplusplus
}
#endif
#endif /* BMB200_H_INCLUDED */
