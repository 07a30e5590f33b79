/* kaminpar_b200 -- C ABI of the ParHIP reader on the device (DESIGN.md §19): a ParHIP binary graph file, or its bytes
 * already in device memory, read into CSR arrays on the GPU, every value checked before a kernel indexes by it.
 *
 * Restates io::parhip::read_graph (kaminpar-io/parhip_parser.cc:580-587) without compression: csr_read (:179-220) and
 * csr_read_deg_buckets (:222-336) with ParHIPHeader (:40-145), on the default build's 32-bit ids and weights. The rule:
 *
 *   Layout. A 24-byte header of three little-endian u64: version, n, m. Then offsets[n+1], adjncy[m], vwgt[n] if
 *     present, adjwgt[m] if present. Version bits (a bit CLEAR means "present" / "64-bit"): 0 edge weights, 1 node
 *     weights, 2 64-bit offsets, 3 64-bit ids, 4 64-bit node weights, 5 64-bit edge weights. Bits above 5 are ignored;
 *     bytes after the last section are ignored.
 *   Offsets. offsets[u] is the byte address of u's adjacency list: xadj[u] = (offsets[u] - base) / id_width with
 *     base = 24 + (n+1) * offset_width (map_edge_offset, :112-114).
 *   Weights. Weights that are present stay present, all-unit weights included (only the METIS reader drops them).
 *   Orderings (NodeOrdering, kaminpar.h:66-71):
 *     NATURAL, DEGREE_BUCKETS   csr_read(sorted = false): the file's arrays;
 *     IMPLICIT_DEGREE_BUCKETS   the same arrays, the graph marked sorted;
 *     EXTERNAL_DEGREE_BUCKETS   csr_read_deg_buckets: new ids are a STABLE sort of the vertices by degree bucket
 *                               (floor(log2 deg) + 1, degree 0 last, permutator.h:105-117); xadj is the prefix sum of
 *                               the degrees in new order; each adjacency list is copied in FORWARD order (unlike
 *                               rearrange_by_degree_buckets, which reverses it) with its targets relabelled through
 *                               old_to_new; weights travel with their vertex and edge; the permutation old_to_new is
 *                               kept and the graph is marked sorted.
 *   KMP_PARHIP_COMPRESS or'ed into the ordering (the compressed read) is KMP_ERR_UNSUPPORTED.
 *
 * Parity domain: the files the reference's default build reads without reading outside its mapping and without a
 * value leaving its types. There the arrays (and the permutation) equal read_graph's bit for bit; a file with 64-bit
 * widths, which that build refuses with exit(1) (ParHIPHeader::validate, :116-138), is read as the same graph written
 * at 32-bit widths. Outside the domain no graph is made: the call returns KMP_ERR_INVALID (KMP_ERR_UNSUPPORTED for
 * TOO_LARGE) and the report holds the FIRST violation in file order: its kind, byte offset, section and the index of
 * the entry within its section. An entry's violation is located at its first byte; at one byte the kind listed first
 * wins.
 *
 *   KMP_PARHIP_TRUNCATED   the file ends before the header or a section does; at the file's length, with the
 *                          section it ends in and its first incomplete entry (read_graph would read past its mapping)
 *   KMP_PARHIP_TOO_LARGE   -> KMP_ERR_UNSUPPORTED: n or m >= 2^31 (the library's 32-bit edge ids hold 2^31 - 1 at
 *                          most; at byte 8 / 16), a 64-bit target >= 2^32 or a 64-bit weight >= 2^31 (narrowing it
 *                          would change it)
 *   KMP_PARHIP_OFFSETS     offsets[0] != base, offsets[u] < offsets[u-1], offsets[u] - base not a multiple of the id
 *                          width, or offsets[n] != base + m * id_width (a kernel would index by the offset)
 *   KMP_PARHIP_NEIGHBOR_OUT_OF_RANGE  a target >= n (the reference indexes by it)
 *   KMP_PARHIP_WEIGHT      a node or edge weight < 1 (the library's weights are positive: the balancers and the
 *                          LP's weight tables assume it)
 *   KMP_PARHIP_TOTAL_WEIGHT the total of the node or of the edge weights does not fit int32 (the graph's totals are
 *                          NodeWeight / EdgeWeight); at the LAST byte of its section, index = n or m
 *
 * Not checked, as in the reference: symmetry, duplicate edges and self-loops. Run kmp_validate_graph_device on the
 * result for those.
 *
 * Device work: element-parallel passes over each section at its width with 16-byte loads; a violation is one 64-bit
 * atomicMin of (offset << 8) | kind, so a valid file issues none; weight totals take one atomic per warp. EXTERNAL
 * reuses the preparation's tile histogram and stable scatter (kmp_prepare.cuh) on the offsets, then copies the edges
 * over tiles of the NEW layout, reading each target from the file's bytes at the file's width: no natural-order CSR
 * is built, but the file's bytes (its natural-order adjncy section among them) stay resident until the edge copy ends,
 * in h's pool for kmp_read_parhip and in the caller's memory for kmp_parse_parhip_device. So the fused read saves no
 * device memory over a read followed by kmp_prepare_graph_device: it needs about the file plus the prepared graph
 * (DESIGN.md §19 measures both). Memory from the handle's pool (the bytes for kmp_read_parhip, the outputs, the scratch, CUB's
 * temporary) is allocated before the first kernel runs: a file that does not fit is KMP_ERR_ALLOC with nothing run.
 *
 * All calls run on h's device, stream and pool and do not touch h's graph, labels or call counter; a handle inside a
 * stepping call is refused (KMP_ERR_INVALID). Same error convention as kaminpar_b200_lp.h (0 = ok,
 * kmp_last_error()). No CPU fallback: every call fails without a GPU.
 */
#ifndef KAMINPAR_B200_PARHIP_H
#define KAMINPAR_B200_PARHIP_H

#include <stddef.h>
#include <stdint.h>

#include "kaminpar_b200_lp.h"
#include "kaminpar_b200_prepare.h"

#ifdef __cplusplus
extern "C" {
#endif

/* orderings: the values of kaminpar::shm::NodeOrdering */
enum {
  KMP_PARHIP_NATURAL = 0,
  KMP_PARHIP_DEGREE_BUCKETS = 1,
  KMP_PARHIP_EXTERNAL_DEGREE_BUCKETS = 2,
  KMP_PARHIP_IMPLICIT_DEGREE_BUCKETS = 3,
  KMP_PARHIP_COMPRESS = 0x100 /* or'ed in: read_graph(compress = true), not supported */
};

enum {
  KMP_PARHIP_OK = 0,
  KMP_PARHIP_TRUNCATED = 1,
  KMP_PARHIP_TOO_LARGE = 2,
  KMP_PARHIP_OFFSETS = 3,
  KMP_PARHIP_NEIGHBOR_OUT_OF_RANGE = 4,
  KMP_PARHIP_WEIGHT = 5,
  KMP_PARHIP_TOTAL_WEIGHT = 6,
  KMP_PARHIP_NUM_KINDS = 7
};

/* the sections of the file, in file order */
enum {
  KMP_PARHIP_SECTION_HEADER = 0,
  KMP_PARHIP_SECTION_OFFSETS = 1,
  KMP_PARHIP_SECTION_ADJNCY = 2,
  KMP_PARHIP_SECTION_VWGT = 3,
  KMP_PARHIP_SECTION_ADJWGT = 4
};

typedef struct kmp_parhip_report {
  int32_t kind;             /* KMP_PARHIP_*: the first violation, KMP_PARHIP_OK for a graph */
  int32_t section;          /* KMP_PARHIP_SECTION_* holding it */
  int32_t has_node_weights; /* version bit 1 clear (as far as the header was read) */
  int32_t has_edge_weights; /* version bit 0 clear */
  int32_t sorted;           /* the graph is marked sorted (IMPLICIT / EXTERNAL) */
  int32_t ordering;         /* the ordering asked for */
  uint64_t version, n, m;   /* the header (0 where the file ends before a field) */
  uint64_t bytes;           /* the file's length */
  uint64_t offset;          /* the first violation: byte offset */
  int64_t index;            /* and entry index within its section (-1: the header) */
  float device_ms;          /* device time of the call (the file's H2D copies included for kmp_read_parhip) */
  uint32_t widths;          /* bytes of offsets, ids, node weights, edge weights: one per byte, lowest first */
} kmp_parhip_report;

/* The graph read: n vertices, m adjacency entries, in h's pool on h's device. */
typedef struct kmp_parhip_graph kmp_parhip_graph;

/* Reads the ParHIP file at `path`. The file is streamed through two pinned host buffers (the METIS reader's), and
 * each pass starts on the entries of a section as soon as their bytes are queued. Refused: NULL h / path / out /
 * report, an unknown ordering: KMP_ERR_INVALID; a file that cannot be opened or read: KMP_ERR_INVALID with
 * report->kind = KMP_PARHIP_OK; a malformed file: see above. *out is set only on success. */
int kmp_read_parhip(kmp_lp_handle *h, const char *path, int ordering, kmp_parhip_graph **out,
                    kmp_parhip_report *report);
/* The same from `len` bytes already on h's device (e.g. a torch uint8 tensor); they are only read. Refused as
 * kmp_parse_metis_device refuses: NULL arguments, d_bytes not 16-byte aligned or not device (or managed) memory of
 * h's device: KMP_ERR_INVALID; len >= 2^56: KMP_ERR_UNSUPPORTED. */
int kmp_parse_parhip_device(kmp_lp_handle *h, const void *d_bytes, uint64_t len, int ordering,
                            kmp_parhip_graph **out, kmp_parhip_report *report);

/* EXTERNAL_DEGREE_BUCKETS straight into a prepared graph: the isolated vertices are the tail, old_to_new is the
 * reference's permutation, and kmp_lp_set_graph_prepared / kmp_prepared_finish take it as it is, so the final
 * partition comes out in the file's vertex ids. The adjacency lists are in forward order (see above). Peak device
 * memory: the file's bytes plus the prepared graph and its scratch (see "Device work"). */
int kmp_read_parhip_prepared(kmp_lp_handle *h, const char *path, kmp_prepared_graph **out,
                             kmp_parhip_report *report);
int kmp_parse_parhip_device_prepared(kmp_lp_handle *h, const void *d_bytes, uint64_t len, kmp_prepared_graph **out,
                                     kmp_parhip_report *report);

uint32_t kmp_parhip_n(const kmp_parhip_graph *g);
uint32_t kmp_parhip_m(const kmp_parhip_graph *g);
int kmp_parhip_sorted(const kmp_parhip_graph *g);
/* The device arrays (NULL for absent weights; old_to_new NULL unless EXTERNAL), valid until kmp_parhip_destroy; they
 * can go straight into kmp_lp_set_graph_device, kmp_validate_graph_device or kmp_prepare_graph_device. */
int kmp_parhip_device_arrays(const kmp_parhip_graph *g, const uint32_t **d_xadj, const uint32_t **d_adjncy,
                             const int32_t **d_vwgt, const int32_t **d_adjwgt, const uint32_t **d_old_to_new);
/* Copies to host arrays of n + 1, m, n, m, n entries; a NULL destination or an absent array copies nothing. */
int kmp_parhip_download(const kmp_parhip_graph *g, uint32_t *xadj, uint32_t *adjncy, int32_t *vwgt, int32_t *adjwgt,
                        uint32_t *old_to_new);
/* Frees the arrays on the reading handle's stream: call it before that handle is destroyed. */
void kmp_parhip_destroy(kmp_parhip_graph *g);

/* The usage of the device memory pool that h and every result of h allocate from (one pool per device, shared by the
 * handles on it), after h's stream is synchronised: *used the bytes in use, *used_high the most in use since the
 * last reset. reset != 0 then restarts the high-water mark at the current use. For measuring the footprint of a call,
 * e.g. the fused EXTERNAL read against a read followed by kmp_prepare_graph_device. Refused: NULL h / used /
 * used_high: KMP_ERR_INVALID. */
int kmp_pool_usage(kmp_lp_handle *h, int reset, uint64_t *used, uint64_t *used_high);

/* One line for the report, NUL-terminated into buf[size] (truncated to fit); returns the full length as snprintf
 * does. A refusal: "<kind> at byte <offset> (<section> entry <index>)"; a graph: "". Pure host code. */
int kmp_parhip_report_message(const kmp_parhip_report *r, char *buf, size_t size);

#ifdef __cplusplus
}
#endif
#endif
