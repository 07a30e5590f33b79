/* kaminpar_b200 -- C ABI of the METIS reader on the device (DESIGN.md §18): a METIS text file, or its bytes already in
 * device memory, parsed into CSR arrays on the GPU, with the first malformed token reported.
 *
 * Restates csr_read (kaminpar-io/metis_parser.cc:158-245) with parse_header (:36-80) and parse_graph (:82-154) on the
 * default build's 32-bit ids and weights. The rule:
 *
 *   Lines. Only ' ' is a space (file_toker.h:73-77). A COMMENT line is a line whose first non-space byte is '%'; comment
 *     lines are skipped before the header and between vertex lines. Every other line is a DATA line, an empty line or a
 *     line of spaces included; the v-th data line after the header is vertex v (so an empty line is an isolated vertex).
 *   Header. `n m [fmt]\n`: tokens of decimal digits separated by spaces, leading spaces allowed. fmt is a decimal number
 *     (011 is 11); only 0, 1, 10 and 11 are supported.
 *   Vertex lines. With node weights (fmt x1x) the line starts with the node weight; then come 1-based targets t, each
 *     stored as t - 1, each followed by its weight with edge weights (fmt xx1). xadj, adjncy, vwgt, adjwgt are then the
 *     arrays of csr_read.
 *   Weights dropped. Node weights are dropped when their total is n, edge weights when their total is 2m (:211-222).
 *   Extra lines. Everything after vertex n-1's line is ignored and never judged. extra_lines is set when the reference
 *     warns "ignorning extra lines": some line after it does not start with '%' in its first byte (:145-153).
 *   Numbers saturate: a token too long for any id or weight is WEIGHT_TOO_LARGE or NEIGHBOR_OUT_OF_RANGE, never wraps.
 *
 * Parity domain: the files the reference parses without reading past the end of the file (beyond peeking one byte
 * after a last line without newline) and without tripping one of its own KASSERTs (plain assert()s without kassert,
 * kaminpar-common/assert.h:22-28). There the arrays equal csr_read's bit for bit. Outside it no graph is made: the
 * call returns KMP_ERR_INVALID (KMP_ERR_UNSUPPORTED where marked) and the report holds the FIRST violation in file
 * order: its kind, byte offset, 1-based line number and vertex (-1 in the header). A violation is located at the first
 * byte of its token; the two MISSING kinds at the end of their line (its '\n', or the file length). At one byte the
 * kind listed first wins. The end-of-file kinds (offset = file length) come after all file-order kinds, in the order
 * listed:
 *
 *   KMP_METIS_EMPTY            the file is empty (the reference's mmap fails, it returns nullopt)
 *   KMP_METIS_HEADER           the header is not `n m [fmt]\n` (a blank line before it, a fourth token, no newline), or
 *                              m > n(n-1)/2 (:69-72); scan_uint's / consume_char's assertion (file_toker.h:89-133)
 *   KMP_METIS_FORMAT           -> KMP_ERR_UNSUPPORTED: fmt is 1xx or another unsupported value (:48-59)
 *   KMP_METIS_TOO_LARGE        -> KMP_ERR_UNSUPPORTED: n >= 2^32 or 2m >= 2^32 (:61-68, 32-bit edge ids); at n or m
 *   KMP_METIS_BAD_BYTE         a byte of a data line that is not a digit, ' ' or '\n' ('\t', '\r', signs, '%' after a
 *                              token)
 *   KMP_METIS_MISSING_NODE_WEIGHT  a data line without tokens while node weights are on
 *   KMP_METIS_MISSING_EDGE_WEIGHT  an odd number of tokens after the node weight while edge weights are on
 *   KMP_METIS_ZERO_WEIGHT      a node or edge weight of 0 (:109, :131)
 *   KMP_METIS_WEIGHT_TOO_LARGE a node or edge weight > 2^31 - 1 (:105-108, :127-130)
 *   KMP_METIS_NEIGHBOR_OUT_OF_RANGE  a target of 0 or above n (:134)
 *   KMP_METIS_SELF_LOOP        a target equal to its own line's vertex (:135)
 *   KMP_METIS_TOO_FEW_LINES    the file ends before vertex n-1's line begins (the reference reads past its mapping:
 *                              this kind is pinned to the rule, not to the reference); vertex = the first missing one
 *   KMP_METIS_EDGE_COUNT       the number of targets is not 2m (:207-208)
 *   KMP_METIS_TOTAL_WEIGHT     the node or the edge weight total does not fit int32 (:224-231)
 *
 * The reader checks neither symmetry nor duplicate edges (the reference's reader does not either): run
 * kmp_validate_graph_device on the result for that.
 *
 * Device work: parallel over the file's bytes in tiles of KMP_METIS_TILE_BYTES, never over lines, so a hub line that
 * spans many tiles costs what its bytes cost. (a) each tile summarises its line-state machine for every entry state,
 * (b) a scan gives every tile its entry state, vertex and token index, (c) each tile re-reads its bytes and writes
 * xadj / adjncy / vwgt / adjwgt by closed form. A violation is one 64-bit atomicMin of (offset, kind): a valid file
 * issues none. Memory from the handle's pool: the bytes (kmp_read_metis), the output arrays, 176 B per tile and CUB's
 * scan temporary, all allocated before the first kernel runs: a file that does not fit is KMP_ERR_ALLOC with no
 * kernel run.
 *
 * Both calls run on h's device, stream and pool; they do not touch h's graph, labels or call counter, so they work on
 * seq_strict and sharded handles alike; a handle inside a stepping call is refused (KMP_ERR_INVALID). Same error
 * convention as kaminpar_b200_lp.h (0 = ok, kmp_last_error()). No CPU fallback: every call fails without a GPU.
 */
#ifndef KAMINPAR_B200_IO_H
#define KAMINPAR_B200_IO_H

#include <stddef.h>
#include <stdint.h>

#include "kaminpar_b200_lp.h"

#ifdef __cplusplus
extern "C" {
#endif

#define KMP_METIS_TILE_BYTES 4096 /* bytes per tile of the device passes, counted from the first byte of the file */

enum {
  KMP_METIS_OK = 0,
  KMP_METIS_EMPTY = 1,
  KMP_METIS_HEADER = 2,
  KMP_METIS_FORMAT = 3,
  KMP_METIS_TOO_LARGE = 4,
  KMP_METIS_BAD_BYTE = 5,
  KMP_METIS_MISSING_NODE_WEIGHT = 6,
  KMP_METIS_MISSING_EDGE_WEIGHT = 7,
  KMP_METIS_ZERO_WEIGHT = 8,
  KMP_METIS_WEIGHT_TOO_LARGE = 9,
  KMP_METIS_NEIGHBOR_OUT_OF_RANGE = 10,
  KMP_METIS_SELF_LOOP = 11,
  KMP_METIS_TOO_FEW_LINES = 12,
  KMP_METIS_EDGE_COUNT = 13,
  KMP_METIS_TOTAL_WEIGHT = 14,
  KMP_METIS_NUM_KINDS = 15
};

typedef struct kmp_metis_report {
  int32_t kind;                 /* KMP_METIS_*: the first violation, KMP_METIS_OK for a graph */
  int32_t has_node_weights;     /* fmt x1x (as far as the header was read) */
  int32_t has_edge_weights;     /* fmt xx1 */
  int32_t node_weights_dropped; /* node weights given, all 1: the graph has none */
  int32_t edge_weights_dropped; /* edge weights given, all 1: the graph has none */
  int32_t extra_lines;          /* the reference's "ignorning extra lines in input file" warning */
  uint64_t n, m;                /* the header's n and m (saturated; 0 before they are read) */
  uint64_t bytes;               /* the file's length */
  uint64_t offset;              /* the first violation: byte offset, */
  uint64_t line;                /* 1-based line number, */
  int64_t vertex;               /* and the vertex whose line holds it (-1: the header) */
  float device_ms;              /* device time of the call (the file's H2D copies included for kmp_read_metis) */
  uint32_t format;              /* the header's fmt (saturated to 2^32 - 1) */
} kmp_metis_report;

/* The parsed graph: n vertices, m = 2 * the header's m adjacency entries, in h's pool on h's device. */
typedef struct kmp_metis_graph kmp_metis_graph;

/* Reads the METIS file at `path`. The file is streamed through two pinned host buffers: reading the next chunk
 * overlaps the copy and summary of the previous one. The header is parsed on the host. Refused: NULL h / path / out /
 * report: KMP_ERR_INVALID; a file that cannot be opened or read: KMP_ERR_INVALID with report->kind = KMP_METIS_OK;
 * a malformed file: see above. *out is set only on success. */
int kmp_read_metis(kmp_lp_handle *h, const char *path, kmp_metis_graph **out, kmp_metis_report *report);
/* The same from `len` bytes already on h's device (e.g. a torch uint8 tensor); they are only read. Refused: NULL h /
 * out / report, or d_bytes NULL with len > 0, or d_bytes not 16-byte aligned, or not device (or managed) memory of
 * h's device: KMP_ERR_INVALID; len >= 2^56: KMP_ERR_UNSUPPORTED. */
int kmp_parse_metis_device(kmp_lp_handle *h, const void *d_bytes, uint64_t len, kmp_metis_graph **out,
                           kmp_metis_report *report);

uint32_t kmp_metis_n(const kmp_metis_graph *g);
uint32_t kmp_metis_m(const kmp_metis_graph *g); /* adjacency entries */
/* The device arrays (NULL for absent or dropped weights), valid until kmp_metis_destroy; they can go straight into
 * kmp_lp_set_graph_device or kmp_prepare_graph_device. */
int kmp_metis_device_arrays(const kmp_metis_graph *g, const uint32_t **d_xadj, const uint32_t **d_adjncy,
                            const int32_t **d_vwgt, const int32_t **d_adjwgt);
/* Copies to host arrays of n + 1, m, n, m entries; a NULL destination or an absent array copies nothing. */
int kmp_metis_download(const kmp_metis_graph *g, uint32_t *xadj, uint32_t *adjncy, int32_t *vwgt, int32_t *adjwgt);
/* Frees the arrays on the reading handle's stream: call it before that handle is destroyed. */
void kmp_metis_destroy(kmp_metis_graph *g);

/* One line for the report, NUL-terminated into buf[size] (truncated to fit); returns the full length as snprintf
 * does. A refusal: "<kind> at byte <offset> (line <line>, vertex <vertex>)"; a graph: the reference's warning line
 * "ignorning extra lines in input file" when extra_lines is set, else "". Pure host code. */
int kmp_metis_report_message(const kmp_metis_report *r, char *buf, size_t size);

#ifdef __cplusplus
}
#endif
#endif
