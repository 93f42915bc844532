/* mgb.h — C ABI of the H100-native `metagraph align` hot path.
 *
 * This is the drop-in boundary: a maintainer of ratschlab/metagraph binds these entry
 * points from a thin `class B200Aligner : public IDBGAligner` (see INTEGRATION.md and
 * metagraph_b200/csrc/b200_aligner.hpp).  Plain pointers and sizes only; no exceptions,
 * STL or torch types cross this boundary.  Every function returns MGB_OK (0) or a
 * negative error code; mgb_last_error() returns a thread-local message.
 *
 * Reference interfaces replaced (paths relative to metagraph/src):
 *   mgb_index_create      <- DBGSuccinct / boss::BOSS query state: W (wavelet_tree), last
 *                            (bit_vector), F (graph/representation/succinct/boss.hpp:499-525),
 *                            optional dummy mask valid_edges_ (dbg_succinct.hpp:195)
 *   mgb_map_to_nodes      <- map_to_nodes_sequentially() (graph/representation/base/
 *                            sequence_graph.cpp:541-551 -> dbg_succinct.cpp:285-305 ->
 *                            boss.cpp:996-1045 BOSS::map_to_edges)
 *   mgb_map_to_nodes_strands  the same for a sequence and its reverse complement at once
 *   mgb_config_check      <- DBGAligner::DBGAligner (graph/alignment/dbg_aligner.cpp:26-60)
 *   mgb_align_batch       <- IDBGAligner::align_batch (graph/alignment/dbg_aligner.hpp:32-33,
 *                            dbg_aligner.cpp:251-355) with Seeder = SuffixSeeder<UniMEMSeeder>,
 *                            Extender = DefaultColumnExtender
 *   mgb_config_t          <- DBGAlignerConfig (graph/alignment/aligner_config.hpp:18-94)
 *   mgb_alignment_t       <- Alignment (graph/alignment/alignment.hpp:132-331)
 *   mgb_boss_build        <- BOSSConstructor / BOSS::Chunk (boss_chunk_construct.cpp:341-462,
 *                            boss_chunk.cpp:33-133); host-side, not part of the timed path
 */
#ifndef MGB_H_
#define MGB_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MGB_OK 0
#define MGB_ERR_INVALID_ARGUMENT (-1)
#define MGB_ERR_CUDA (-2)
#define MGB_ERR_BAD_CONFIG (-3)   /* reference: std::runtime_error in DBGAligner ctor (dbg_aligner.cpp:55-56) */
#define MGB_ERR_UNSUPPORTED (-4)  /* a configuration or graph the kernels do not serve (chaining, labels, ...) */
#define MGB_ERR_OVERFLOW (-5)     /* a read exceeded the largest per-read work arena */
#define MGB_ERR_NO_DEVICE (-6)
#define MGB_ERR_NO_MEMORY (-7)    /* host allocation failed (index construction) */

#define MGB_ALPHABET_DNA 0      /* "$ACGT", sigma = 5 (kmer/alphabets.hpp:64-79) */
#define MGB_ALPHABET_PROTEIN 1  /* "$ABCDEFGHIJKLMNOPQRSTUVWYZX", sigma = 27 (kmer/alphabets.hpp:29-38) */

/* Cigar::Operator (graph/alignment/aligner_cigar.hpp:18-25); printed as "SX=DIG" */
#define MGB_OP_CLIPPED 0
#define MGB_OP_MISMATCH 1
#define MGB_OP_MATCH 2
#define MGB_OP_DELETION 3
#define MGB_OP_INSERTION 4
#define MGB_OP_NODE_INSERTION 5

typedef struct mgb_index mgb_index_t;
typedef struct mgb_results mgb_results_t;

/* DBGAlignerConfig (aligner_config.hpp:23-61). Penalties are negative as in the struct
 * (cli/align.cpp:33-69 negates the positive CLI values). */
typedef struct mgb_config {
    uint64_t num_alternative_paths;   /* 1..32 (--align-alternative-alignments); larger: MGB_ERR_UNSUPPORTED */
    uint64_t min_seed_length;
    uint64_t max_seed_length;
    uint64_t max_num_seeds_per_locus;
    int32_t min_cell_score;
    int32_t min_path_score;
    int32_t xdrop;
    int32_t reserved0;
    double min_exact_match;
    double max_nodes_per_seq_char;
    double max_ram_per_alignment;
    double rel_score_cutoff;
    int8_t gap_opening_penalty;
    int8_t gap_extension_penalty;
    int8_t left_end_bonus;
    int8_t right_end_bonus;
    uint8_t forward_and_reverse_complement;
    uint8_t global_xdrop;
    uint8_t allow_left_trim;
    uint8_t no_backtrack;
    uint8_t seed_complexity_filter; /* sdust(T=20, W=64) on seed windows, restated from its definition (library not vendored) */
    /* What mgb_alignment_t::nodes carries (not a DBGAlignerConfig field): MGB_NODES_U64 = the node path (default),
     * MGB_NODES_NONE = nothing (nodes == NULL, num_nodes still set) for consumers that only print alignments
     * (the TSV branch of cli/align.cpp:254-307 never reads Alignment::get_nodes()): the node ids are 4/5 of the
     * bytes a 150 bp alignment brings back from the device. */
    uint8_t result_nodes;
    /* 1 = never take the exact-path shortcut: when every k-mer of a strand is in the graph, the seed at query
     * position 0 extends, provably, to the whole read matched along those nodes (DESIGN.md "Exact-path shortcut":
     * conditions on the scores, proof, what the reference does instead); the kernel then writes that alignment
     * without running the extension. Results are identical either way; the switch exists for measurements. */
    uint8_t no_exact_path_shortcut;
    uint8_t reserved1[5];
    int8_t score_matrix[128][128];
} mgb_config_t;
enum { MGB_NODES_U64 = 0, MGB_NODES_NONE = 1 };

/* One alignment of one read (Alignment, alignment.hpp:323-331). Pointers reference memory
 * owned by the enclosing mgb_results_t. */
typedef struct mgb_alignment {
    uint32_t read_index;
    uint8_t orientation;       /* 1: the reverse complement of the read was aligned */
    uint8_t pad[3];
    int32_t score;
    uint32_t offset;           /* chars discarded from the first node's prefix */
    uint32_t query_begin;      /* == leading clipping; query_view = strand[query_begin, +query_len) */
    uint32_t query_len;
    uint32_t num_nodes;
    uint32_t sequence_len;
    uint32_t num_cigar_ops;
    uint32_t reserved;
    const uint64_t *nodes;     /* DBG node ids == BOSS edge indexes */
    const char *sequence;      /* spelling of the path (not NUL-terminated) */
    const uint32_t *cigar;     /* (len << 3) | op, clipping included */
} mgb_alignment_t;

/* Per-batch counters (dbg_aligner.cpp:341-351 trace line; dp_cells is the GCUPS numerator,
 * SURVEY 8d). */
typedef struct mgb_stats {
    uint64_t num_seeds;
    uint64_t num_extensions;
    uint64_t num_explored_nodes;
    uint64_t dp_cells;
    uint64_t dp_columns;
    uint64_t num_reads_retried;   /* reads re-run with a larger work arena */
    double seed_kernel_ms;        /* device time of the seeding kernel(s) */
    double align_kernel_ms;       /* device time of the extension kernel(s) */
    double h2d_ms, d2h_ms;
    uint64_t h2d_bytes, d2h_bytes;
    uint64_t kernel_launches;
} mgb_stats_t;

const char* mgb_last_error(void);
int mgb_device_count(void);

/* ---- index -------------------------------------------------------------------------- */

/* Uploads a BOSS table into HBM in the flat block layout described in DESIGN.md.
 *   W[0..n]     edge labels incl. the position-0 placeholder, values in [0, 2*sigma)
 *   last[0..n]  0/1 bytes
 *   F[sigma]    boss F array
 *   valid       optional 0/1 bytes (dummy-k-mer mask); NULL = mask dropped, which is what
 *               `metagraph align` does (cli/align.cpp:335-339)
 *   k           DBG k-mer length (BOSS node length + 1)
 *   suffix_len  length of the indexed suffix ranges (boss.hpp:516-525); 0 = choose */
int mgb_index_create(const uint8_t *W, const uint8_t *last, uint64_t n_plus_1,
                     const uint64_t *F, const uint8_t *valid, uint32_t k, int alphabet,
                     uint32_t suffix_len, int device, mgb_index_t **out);
/* DeBruijnGraph::get_mode() of the graph (sequence_graph.hpp:160): 0 = BASIC (default), 1 = CANONICAL (built with
 * --mode canonical: the graph holds the reverse complement of every k-mer; dbg_aligner.cpp:224-226, 646-722).
 * 2 = PRIMARY (built with --mode primary: one k-mer of every reverse-complement pair): the index answers with the
 * semantics of the CanonicalDBG wrapper `metagraph align` puts around such graphs (canonical_dbg.cpp): node ids
 * above mgb_index_num_edges() denote reverse complements. The first call builds two 4-byte-per-edge tables on the
 * device; mgb_map_to_nodes then follows CanonicalDBG::map_to_nodes_sequentially (both strands, canonical_dbg.cpp:55-146).
 * Set the mode once, right after mgb_index_create and before the index is shared between threads. */
int mgb_index_set_mode(mgb_index_t *index, int mode);
void mgb_index_destroy(mgb_index_t *index);
/* A copy of src on `device` (src's own device allowed), made device to device: no host build, no build kernels.
 * The graph mode and the tables mgb_index_set_mode built come along. The replica is independent of src: either may
 * be destroyed first, and both may be used from several threads at once. Table for table, the replica is what
 * mgb_index_create would build on `device` at that moment: the k-mer hash index, the path layout and its two leaner
 * copies (DESIGN.md §4) follow the build's free-memory rules and knobs on that device, so a replica may leave out a
 * table its source holds, never the reverse; results do not depend on these tables. A bad ordinal or a null
 * argument: MGB_ERR_INVALID_ARGUMENT; a failed allocation or copy: MGB_ERR_CUDA, and nothing stays allocated. */
int mgb_index_replicate(const mgb_index_t *src, int device, mgb_index_t **out);
uint64_t mgb_index_num_edges(const mgb_index_t *index);
uint64_t mgb_index_device_bytes(const mgb_index_t *index);
uint32_t mgb_index_k(const mgb_index_t *index);

/* ---- hot path ------------------------------------------------------------------------ */

/* Default configs. mgb_config_init = DBGAlignerConfig{} + dna_scoring_matrix(2,-1,-2)
 * (what the reference unit tests use); mgb_config_init_cli = `metagraph align` defaults
 * (cli/config/config.hpp:114-145) for a graph with k-mer length k: DNA match 2 / mismatch -3, protein
 * BLOSUM62 and forward strand only. seed_complexity_filter is left 0 (the CLI turns it on; its sdust
 * dependency is restated here, see DESIGN.md) — set it to 1 for flag-free `metagraph align` behaviour. */
void mgb_config_init(mgb_config_t *config);
void mgb_config_init_cli(mgb_config_t *config, uint32_t k, int alphabet);

/* What the DBGAligner constructor checks (dbg_aligner.cpp:37-60: seed-length normalisation, check_config_scores ->
 * std::runtime_error("Error: sum of min_cell_score and lowest penalty too low.")) plus what this build does not serve:
 * MGB_OK, MGB_ERR_BAD_CONFIG or MGB_ERR_UNSUPPORTED with the text in mgb_last_error(). mgb_align_batch makes the same
 * check; this entry point lets a binding fail at construction time, as the reference does. No device work. */
int mgb_config_check(const mgb_index_t *index, const mgb_config_t *config);

/* Exact seeding only: node ids of all k-mers of each sequence (0 = not in graph), forward
 * strand. seqs: concatenated characters, offsets[n_seqs + 1]. out_nodes must hold
 * sum(max(0, len_i - k + 1)) entries, laid out consecutively per sequence. */
int mgb_map_to_nodes(const mgb_index_t *index, const char *seqs, const uint64_t *offsets,
                     uint32_t n_seqs, uint64_t *out_nodes);

/* Exact seeding of both raw strands, in any mode: out_fwd receives the node ids of the k-mers of each sequence
 * and out_rc those of its reverse complement, each laid out as out_nodes of mgb_map_to_nodes. Ids are the stored
 * graph's own (BOSS edges): there is no PRIMARY-mode merge of the two strands. DNA graphs only. */
int mgb_map_to_nodes_strands(const mgb_index_t *index, const char *seqs, const uint64_t *offsets,
                             uint32_t n_seqs, uint64_t *out_fwd, uint64_t *out_rc);

/* Full seed-and-extend of a batch of reads; results in input order. */
int mgb_align_batch(const mgb_index_t *index, const mgb_config_t *config, const char *seqs,
                    const uint64_t *offsets, uint32_t n_reads, mgb_results_t **out);

/* The same seed-and-extend as mgb_align_batch, delivered as the text `metagraph align` prints (cli/align.cpp:254-307),
 * rendered on the device: the records never leave it, only the text is downloaded.
 *   MGB_TEXT_TSV   one line per read: header, upper-cased query (bytes >= 0x80 as 0x7F), then per alignment strand,
 *                  path sequence, score, matches, CIGAR and offset; an unaligned read gets "*\t*\t{min_path_score}\t*\t*\t*"
 *   MGB_TEXT_JSON  one Alignment::to_json record per alignment (one empty record for an unaligned read), keys sorted,
 *                  no whitespace, node ids included
 * Every line ends with '\n'; reads in input order. headers: concatenated header bytes, header_offsets[n_reads + 1]
 * (copied as they are; in JSON only '"', '\\' and bytes below 0x20 are escaped). The bytes are those of
 * format_alignment / format_alignment_json in metagraph_b200/aligner.py. The result set answers mgb_results_text,
 * mgb_results_num_reads, mgb_results_read_range (counts), mgb_results_num_alignments and mgb_results_stats;
 * mgb_results_alignments returns NULL and mgb_results_export fails. An unknown format: MGB_ERR_INVALID_ARGUMENT. */
enum { MGB_TEXT_TSV = 1, MGB_TEXT_JSON = 2 };
int mgb_align_batch_text(const mgb_index_t *index, const mgb_config_t *config, const char *seqs,
                         const uint64_t *offsets, const char *headers, const uint64_t *header_offsets,
                         uint32_t n_reads, int format, mgb_results_t **out);
/* `metagraph align FILE` from the bytes of the file: parses the complete FASTA/FASTQ records of buf[0, bytes) as
 * kseq_read does (seq_io/sequence_io.hpp:349-438), aligns them and renders their text as mgb_align_batch_text does.
 * buf starts at a record start; at_eof = 1 for the last chunk of a file. *consumed = bytes up to the end of the last
 * complete record: the caller keeps buf[*consumed, bytes) for the front of the next chunk, and grows its buffer when
 * *consumed is 0 and at_eof is 0. *ended = 1 when a malformed record ended the input as it ends FastaParser's
 * iteration: the caller reads no more of this file. comment_delim: NULL = the header is the name only, otherwise
 * `--header-comment-delim` (cli/align.cpp:430-435). flags: MGB_FASTX_FWD_AND_REVERSE = `--fwd-and-reverse`, every
 * record followed by its reverse complement under the same header. format: MGB_TEXT_TSV / MGB_TEXT_JSON.
 * The records are parsed on the device when the chunk is a FASTA chunk without '+' lines or a 4-line FASTQ chunk and
 * is shorter than 4 GiB; other chunks are parsed on the host. Either way the bytes are the same. */
enum { MGB_FASTX_FWD_AND_REVERSE = 1 };
int mgb_align_fastx_text(const mgb_index_t *index, const mgb_config_t *config, const char *buf, uint64_t bytes,
                         int at_eof, const char *comment_delim, int flags, int format,
                         uint64_t *consumed, int *ended, mgb_results_t **out);
/* mgb_align_fastx_text in two steps, so that a caller learns where a chunk's records end long before they are
 * aligned, and can hand the rest of its buffer on while the device aligns. mgb_fastx_stage parses the complete records
 * of buf[0, bytes) as mgb_align_fastx_text does (on the device, or on the host for a chunk the device route refuses)
 * and returns once *consumed and *ended are known. The records stay on index's device (or in host memory for a
 * refused chunk); buf may be reused as soon as this returns. A staged batch holds one of the index's working-memory
 * sets until it is aligned or freed. mgb_align_fastx_batch_text aligns and renders a staged batch as
 * mgb_align_fastx_text would have, result stats included; the batch is consumed, also on error. A batch staged on
 * another index: MGB_ERR_INVALID_ARGUMENT. mgb_fastx_batch_free frees a batch that will not be aligned (NULL: no-op). */
typedef struct mgb_fastx_batch mgb_fastx_batch_t;
int mgb_fastx_stage(const mgb_index_t *index, const char *buf, uint64_t bytes, int at_eof, const char *comment_delim,
                    int flags, uint64_t *consumed, int *ended, mgb_fastx_batch_t **out);
int mgb_align_fastx_batch_text(const mgb_index_t *index, const mgb_config_t *config, mgb_fastx_batch_t *batch,
                               int format, mgb_results_t **out);
void mgb_fastx_batch_free(mgb_fastx_batch_t *batch);
/* mgb_fastx_stage for BGZF input (the block gzip of htslib's bgzip: gzip members of at most 64 KiB of text whose header
 * carries the member's size). Stages the text `head` (carried over from the previous chunk, host memory) followed by
 * the text of the complete BGZF blocks at the start of cbuf, inflated on index's device, until their text reaches
 * max_text. Returns as mgb_fastx_stage does, *consumed and *ended over head + inflated text. *c_consumed: compressed
 * bytes of the blocks taken. *c_refused = 1: the member at *c_consumed is not served by the device route (not a BGZF
 * block, its inflate, CRC32 or ISIZE check failed, or it is cut off by the end of the input, c_eof); blocks after it
 * are not taken. The records are parsed with at_eof = c_eof && *c_consumed == cbytes && !*c_refused. The text after
 * *consumed stays with the batch (mgb_fastx_batch_tail). The batch is aligned by mgb_align_fastx_batch_text; its
 * h2d_bytes count the compressed bytes uploaded. */
int mgb_fastx_stage_bgzf(const mgb_index_t *index, const char *head, uint64_t head_bytes, const uint8_t *cbuf,
                         uint64_t cbytes, int c_eof, uint64_t max_text, const char *comment_delim, int flags,
                         uint64_t *c_consumed, int *c_refused, uint64_t *consumed, int *ended,
                         mgb_fastx_batch_t **out);
/* text[consumed, end) of a batch staged by mgb_fastx_stage_bgzf or mgb_fastx_stage_gzip, owned by the batch (valid until it is aligned or
 * freed); empty for a batch of mgb_fastx_stage */
int mgb_fastx_batch_tail(const mgb_fastx_batch_t *batch, const char **tail, uint64_t *bytes);
/* Diagnostic entry, as mgb_fastx_parse is: the complete BGZF blocks of cbuf inflated on index's device and downloaded
 * into out (MGB_ERR_OVERFLOW if they do not fit). *n_blocks: blocks inflated; *c_consumed and *refused as in
 * mgb_fastx_stage_bgzf. */
int mgb_bgzf_inflate(const mgb_index_t *index, const uint8_t *cbuf, uint64_t cbytes, int c_eof, char *out,
                     uint64_t out_cap, uint64_t *out_bytes, uint64_t *c_consumed, uint64_t *n_blocks, int *refused);
/* Plain gzip input (RFC 1952 members, as gzip and pigz write them). A stream holds, in host memory, where the next
 * stage starts and the state of the member it is in: the bit position, the member's last 32 KiB of text and its running
 * CRC32 and length. Any device may stage the next part of a stream. mgb_gzip_stream_state: *in_member = 1 while the
 * stream is inside a member, and *member_text = that member's text staged so far (0 between members). */
typedef struct mgb_gzip_stream mgb_gzip_stream_t;
int mgb_gzip_stream_create(mgb_gzip_stream_t **out);
void mgb_gzip_stream_free(mgb_gzip_stream_t *stream);
int mgb_gzip_stream_state(const mgb_gzip_stream_t *stream, int *in_member, uint64_t *member_text);
/* A stream as one relocatable byte block, so that another process may stage its next part (the `--distributed`
 * command passes it on with the token): its bit position, 32 KiB window, running CRC32 and length, and whether it is
 * inside a member. mgb_gzip_stream_export writes it into caller memory of at least mgb_gzip_stream_export_bytes bytes;
 * mgb_gzip_stream_import rebuilds a stream from such a block (free it with mgb_gzip_stream_free). A stream is not tied
 * to an index or a device. */
uint64_t mgb_gzip_stream_export_bytes(const mgb_gzip_stream_t *stream);
int mgb_gzip_stream_export(const mgb_gzip_stream_t *stream, void *dst, uint64_t capacity);
int mgb_gzip_stream_import(const void *block, uint64_t bytes, mgb_gzip_stream_t **out);
/* mgb_fastx_stage_bgzf for plain gzip input. cbuf holds the stream's next bytes (its first byte partly decoded when
 * the stream is inside a member). Stages `head` followed by the text of the stream, inflated on index's device, up to
 * the last DEFLATE block boundary it confirmed once the text reaches max_text, or up to the member's end, where the
 * CRC32 and ISIZE are checked. A stage never runs past a member's end; the next member's header is read by the next
 * call. *c_consumed: whole bytes of cbuf taken (the stream keeps the bit offset into the next one). *c_refused = 1: the
 * stream at this point is left to the caller, and nothing of it was staged in this call (the stream is unchanged): the
 * member header is not one this route serves (not gzip, not DEFLATE, reserved flags), the bytes after a member are
 * not a member, the stream is invalid, a trailer does not match, the input ends inside a member (c_eof), or a member's
 * first stage could not be split (stored or fixed-Huffman blocks only). *c_consumed = 0 without a refusal: the call
 * needs more compressed bytes to make progress. Records are parsed with at_eof = c_eof, every byte taken and the
 * stream between members. */
int mgb_fastx_stage_gzip(const mgb_index_t *index, mgb_gzip_stream_t *stream, const char *head, uint64_t head_bytes,
                         const uint8_t *cbuf, uint64_t cbytes, int c_eof, uint64_t max_text, const char *comment_delim,
                         int flags, uint64_t *c_consumed, int *c_refused, uint64_t *consumed, int *ended,
                         mgb_fastx_batch_t **out);
/* Diagnostic entry: the gzip members of cbuf inflated on index's device, stage after stage, until the input ends or a
 * stage refuses (*refused, *c_consumed as in mgb_fastx_stage_gzip). sub_bytes: compressed bytes per sub-range (0: the
 * default). cands (n_cands bit offsets in cbuf, or NULL): the candidate block starts, in place of the finder's. counts:
 * sub-ranges, candidates found at or before the end of the text they staged, and candidates confirmed, over all
 * stages. *out_bytes: the text's length, also when it does not fit out_cap (MGB_ERR_OVERFLOW). */
int mgb_gzip_inflate(const mgb_index_t *index, const uint8_t *cbuf, uint64_t cbytes, int c_eof, uint64_t sub_bytes,
                     const uint64_t *cands, uint64_t n_cands, char *out, uint64_t out_cap, uint64_t *out_bytes,
                     uint64_t *c_consumed, int *refused, uint64_t *counts);
/* Diagnostic entry, not needed to align files: the reads and headers mgb_align_fastx_text aligns for the same
 * arguments, without aligning them, so that the device parser can be checked against the host restatement and either
 * parser can be timed on its own. device_route = 1:
 * parsed as mgb_align_fastx_text parses them on index's device; *refused = 1 when the chunk left the device route and
 * the host restatement parsed it. device_route = 0: the host restatement (index may be NULL). The arrays are the
 * caller's: seqs of max_seq_bytes, names of max_name_bytes, offsets and name_offsets of max_records + 1 entries;
 * MGB_ERR_OVERFLOW when the records do not fit. */
int mgb_fastx_parse(const mgb_index_t *index, const char *buf, uint64_t bytes, int at_eof, const char *comment_delim,
                    int flags, int device_route, char *seqs, uint64_t max_seq_bytes, uint64_t *offsets, char *names,
                    uint64_t max_name_bytes, uint64_t *name_offsets, uint64_t max_records, uint64_t *n_records,
                    uint64_t *consumed, int *ended, int *refused);
/* ---- device-resident batches ---------------------------------------------------------- */

/* The same seed-and-extend as mgb_align_batch over n_reads reads that already sit in device memory on index's device
 * (a basecaller's output, a torch tensor); the results stay on the device as columns (mgb_device_results_write).
 *   stream   cudaStream_t of the caller (NULL = the legacy default stream). Before reading d_seqs or offsets the call
 *            makes its own stream wait on an event recorded on `stream`, so reads produced by work still queued there
 *            may be passed.
 *   d_seqs   device memory on index's device (checked with cudaPointerGetAttributes: a host pointer or another device's
 *            pointer is MGB_ERR_INVALID_ARGUMENT); read r is d_seqs[offsets[r], offsets[r + 1]). It may start at any
 *            byte and end at the end of its allocation: the route first copies the reads device to device into the
 *            batch's own 16-byte-aligned buffer with 64 bytes of padding, and no kernel reads the caller's buffer.
 *            NULL is accepted when the reads hold no characters.
 *   offsets  [n_reads + 1], host memory, or device memory on index's device when offsets_on_device = 1. Device offsets
 *            are downloaded once (8 bytes per read). Then they are checked as mgb_align_batch checks them
 *            (non-decreasing, read length): MGB_ERR_INVALID_ARGUMENT.
 * A configuration fails exactly as it fails in mgb_align_batch, with the same code and text. The call blocks the host
 * until the align passes are done, as mgb_align_batch does (retry passes are decided on the host); per pass only a
 * 48-byte summary comes down, plus 4 bytes per read that overflowed its arena. The whole batch runs as one piece on
 * one stream. The handle holds one of the index's working-memory sets, as a staged FASTX batch does, until it is
 * freed; a batch too large for device memory fails with MGB_ERR_CUDA. */
typedef struct mgb_device_results mgb_device_results_t;
int mgb_align_batch_device(const mgb_index_t *index, const mgb_config_t *config, const char *d_seqs,
                           const uint64_t *offsets, int offsets_on_device, uint32_t n_reads, void *stream,
                           mgb_device_results_t **out);
/* Element counts of the columns: n_reads, alignments, sequence bytes, CIGAR ops and node ids (0 with MGB_NODES_NONE). */
typedef struct { uint64_t n_reads, n_alignments, sequence_bytes, cigar_ops, nodes; } mgb_device_sizes_t;
int mgb_device_results_sizes(const mgb_device_results_t *res, mgb_device_sizes_t *sizes);
/* The counters of the batch; num_seeds .. num_reads_retried equal mgb_align_batch's for the same reads. h2d_bytes and
 * d2h_bytes count what crossed PCIe: up, the offsets and their k-mer offsets (16 bytes per read) and each pass's read
 * list (4 bytes per read; pass 0's only when no read was answered before it); down, device offsets, 48 bytes per pass,
 * each retry list and 32 bytes of totals. */
const mgb_stats_t *mgb_device_results_stats(const mgb_device_results_t *res);
/* Caller-allocated device arrays on index's device, sized from mgb_device_sizes_t. Alignment i has the mgb_alignment_t
 * fields of the i-th record mgb_align_batch returns for the same reads, in the same order. */
typedef struct {
    uint64_t *read_first;        /* [n_reads + 1]: the alignments of read r are [read_first[r], read_first[r + 1]) */
    uint32_t *read_index;        /* [n_alignments] each: the read's position in the batch, then the mgb_alignment_t fields */
    uint8_t *orientation;
    int32_t *score;
    uint32_t *offset, *query_begin, *query_len, *num_nodes, *sequence_len, *num_cigar_ops;
    char *sequence;              /* [sequence_bytes]: the path spellings, back to back */
    uint64_t *sequence_offsets;  /* [n_alignments + 1] */
    uint32_t *cigar;             /* [cigar_ops]: (len << 3) | op */
    uint64_t *cigar_offsets;     /* [n_alignments + 1] */
    uint64_t *nodes;             /* [nodes]: node ids (none with MGB_NODES_NONE) */
    uint64_t *node_offsets;      /* [n_alignments + 1] */
} mgb_device_columns_t;
/* Enqueues the column writes on `stream` (cudaStream_t, NULL = legacy default) and returns without synchronising. A
 * NULL pointer for an array with at least one element: MGB_ERR_INVALID_ARGUMENT. May be called more than once. */
int mgb_device_results_write(const mgb_device_results_t *res, const mgb_device_columns_t *dst, void *stream);
/* Waits for the last mgb_device_results_write, then returns the working memory to the index. NULL is a no-op. */
void mgb_device_results_free(mgb_device_results_t *res);

/* The text block of a result set of mgb_align_batch_text (owned by it); MGB_ERR_INVALID_ARGUMENT for a record set. */
int mgb_results_text(const mgb_results_t *results, const char **text, uint64_t *bytes);

/* A batch of >= 128k reads is split into up to 8 contiguous pieces that run on two streams, so the
 * download and unpacking of one piece overlap the kernels of the next (reads are independent,
 * dbg_aligner.cpp:251-355). max_pieces caps the split; 1 = one piece (device timers in mgb_stats_t
 * then do not overlap), 0 = automatic (default). Process-wide. */
void mgb_set_pipeline_pieces(uint32_t max_pieces);
/* Host threads for the unpacking of results (mgb_align_batch, mgb_results_export / import): launchers such as
 * torchrun start every rank with OMP_NUM_THREADS=1; a rank that owns cores/ranks of them says so here. Process-wide.
 * The library never uses more than 16 threads per call for this work whatever the setting (the loops are short). */
void mgb_set_host_threads(int num_threads);

uint32_t mgb_results_num_reads(const mgb_results_t *results);
/* alignments of read i are [first, first + count) in mgb_results_alignments() */
void mgb_results_read_range(const mgb_results_t *results, uint32_t read, uint64_t *first,
                            uint32_t *count);
uint64_t mgb_results_num_alignments(const mgb_results_t *results);
const mgb_alignment_t* mgb_results_alignments(const mgb_results_t *results);
const mgb_stats_t* mgb_results_stats(const mgb_results_t *results);
void mgb_results_free(mgb_results_t *results);

/* Multi-GPU: reads shard across ranks (one process per GPU, SURVEY 8e; dbg_aligner.cpp:263-354 keeps no state
 * between reads) and rank 0 collects the per-rank results. mgb_results_export writes a result set as one
 * relocatable byte block (the records as the kernel packed them, no pointers) into caller memory -- e.g. a pinned
 * buffer handed to ncclSend; mgb_results_import rebuilds a result set from such a block on the receiving rank,
 * with read_index_base added to the read indexes (the shard's first read). */
uint64_t mgb_results_export_bytes(const mgb_results_t *results);
int mgb_results_export(const mgb_results_t *results, void *dst, uint64_t capacity);
int mgb_results_import(const void *block, uint64_t bytes, uint32_t read_index_base, mgb_results_t **out);

/* ---- host-side construction (index build, untimed) ------------------------------------ */

/* Builds BOSS arrays from sequences (batch construction incl. dummy edges). Caller frees
 * with mgb_boss_free. force_source_dummies mimics BOSS::add_sequence leftovers. (k+1)-mers are packed into 128-bit
 * keys, 256-bit ones beyond (DNA: k <= 85, protein: k <= 51; larger k: MGB_ERR_UNSUPPORTED). */
typedef struct mgb_boss {
    uint64_t n_plus_1;
    uint8_t *W;
    uint8_t *last;
    uint64_t F[32];
    uint32_t k;        /* DBG k */
    int32_t alphabet;
} mgb_boss_t;
int mgb_boss_build(const char *seqs, const uint64_t *offsets, uint32_t n_seqs, uint32_t k,
                   int alphabet, int force_source_dummies, int num_threads, mgb_boss_t *out);
/* Text for the last failed mgb_boss_build() on this thread ("" after a success). */
const char* mgb_boss_last_error(void);
void mgb_boss_free(mgb_boss_t *boss);
/* Dummy-k-mer mask as DBGSuccinct::mask_dummy_kmers computes it (dbg_succinct.cpp:917-932);
 * valid must hold n_plus_1 bytes. */
int mgb_boss_mask_dummy(const mgb_boss_t *boss, uint8_t *valid);

/* Reads a graph file written by the reference (`.dbg`: DBGSuccinct::serialize, dbg_succinct.cpp:690-803 ->
 * BOSS::serialize, boss.cpp:262-277) into plain BOSS arrays for mgb_index_create(). States SMALL and STAT
 * (boss.hpp:325); DYN / FAST files are refused. *mode = DeBruijnGraph::Mode (0 BASIC, 1 CANONICAL,
 * 2 PRIMARY; pass it to mgb_index_set_mode), *state = BOSS::State. The suffix
 * range index and the optional .edgemask file are not read. Free with mgb_boss_free(). On failure returns
 * MGB_ERR_INVALID_ARGUMENT and mgb_dbg_last_error() describes why. */
int mgb_dbg_load(const char *path, mgb_boss_t *out, int *mode, int *state);
/* The file's own index of suffix ranges (BOSS::serialize_suffix_ranges / load_suffix_ranges, boss.cpp:396-426; what
 * BOSS::get_initial_range consults, boss.hpp:638-664), decoded: *suffix_len = indexed suffix length s (0: the file has
 * none), ranges[2 i], ranges[2 i + 1] = first edge and one past the last edge of the nodes whose last s characters
 * are the i-th s-mer (index = sum over positions p of (code_p - 1) (sigma - 1)^p; an empty range has both equal).
 * mgb_index_create builds its own, deeper table on the device and does not need this one: the entry point exists for
 * callers that keep using the file's table and for checking one against the other. Free with
 * mgb_dbg_free_suffix_ranges(). */
int mgb_dbg_load_suffix_ranges(const char *path, uint32_t *suffix_len, uint64_t **ranges, uint64_t *n_ranges);
void mgb_dbg_free_suffix_ranges(uint64_t *ranges);
const char* mgb_dbg_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* MGB_H_ */
