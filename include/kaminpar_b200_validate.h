/* kaminpar_b200 -- C ABI of graph validation on the device (DESIGN.md §17): is a caller's CSR graph what KaMinPar
 * requires (undirected, no self-loops, every reverse edge with the same weight), and if not, where does it first fail.
 *
 * Restates, for CSR graphs with 32-bit ids / weights (the default build types, kaminpar.h:32-57):
 *
 *   debug::validate_graph(n, xadj, adjncy, vwgt, adjwgt, check_undirected = true, num_pseudo_nodes = 0)
 *                              kaminpar-shm/datastructures/csr_graph.cc:266-356 (what KaMinPar::borrow_and_mutate_graph
 *                              and copy_graph assert, kaminpar.cc:174, :215)
 *   the multi-edge check that validate_undirected_graph intends (graphutils/graph_validator.cc:33-85, the CLI's
 *                              --validate), on the sorted row
 *
 * The rule. The input is n, m, xadj[n+1], adjncy[m] and adjwgt[m] or NULL; the report is a pure function of them.
 * The checks run in this order and the FIRST violation is reported:
 *   1. shape (the analogue of the reference's array-size checks, csr_graph.cc:275-290):
 *        KMP_GRAPH_XADJ_START  xadj[0] != 0;        KMP_GRAPH_XADJ_END  xadj[n] != m;
 *   2. KMP_GRAPH_XADJ_DECREASING at the smallest u with xadj[u] > xadj[u+1] (:292-297).
 *      Once 1 or 2 fails, no row is read.
 *   3. every edge e = (u, v) in ascending e (the reference's (u, e) loop order), under the first kind that applies:
 *        KMP_GRAPH_NEIGHBOR_OUT_OF_GRAPH  v >= n;
 *        KMP_GRAPH_SELF_LOOP              v == u;
 *      otherwise, with p the FIRST position of u in v's row (input order) and q the first position in v's row whose
 *      target is >= n:
 *        KMP_GRAPH_NEIGHBOR_OF_NEIGHBOR_OUT_OF_GRAPH  q exists and q < p (or u is absent), reported with q, adjncy[q];
 *        KMP_GRAPH_MISSING_REVERSE                    p does not exist;
 *        KMP_GRAPH_WEIGHT_MISMATCH                    edge weights and adjwgt[e] != adjwgt[p], reported with p.
 *      This is csr_graph.cc:299-353 exactly; its e >= m checks cannot fire once 1-2 pass.
 *   4. duplicate neighbours, beside the verdict and not part of it (KaMinPar's API accepts multi-edges): the number of
 *      edges whose target appeared earlier in the same row, and the first such (u, e): the smallest u that has any
 *      and in it the smallest such position e.
 *
 * Parity domain: for every input of the declared sizes, `kind` and the first violation's fields equal what
 * debug::validate_graph returns and prints, where the reference can see the violation at all (it has no analogue of
 * XADJ_START and reads m from xadj[n]). `valid && duplicates == 0` equals validate_undirected_graph's verdict on graphs
 * with in-range targets, no self-loops and duplicate targets (if any) next to each other in their row: that validator
 * compares neighbours in input order, so it passes a row such as [a, b, a], which this report flags as a duplicate.
 * Not checked (the reference does not check them either): weight signs, total-weight overflow, vwgt.
 *
 * Safety: the check is safe on ANY arrays of the declared sizes. No row is indexed by xadj before 1-2 have passed
 * (one host wait), and no target is used as an index before it is compared with n.
 *
 * Cost: device scratch from the handle's pool of 12 B per edge (sorted targets, positions and their sorted copy), 4 B
 * per vertex (the first target >= n per row), 4 B per 2048 edges, plus CUB's segmented-sort temporary (on the
 * handle's scratch); a host input is first copied to the device (4 B per vertex, 4 or 8 B per edge). All of it is
 * allocated before the first kernel runs.
 *
 * The call runs on h's device, stream and pool. It does not touch h's graph, labels, weights or call counter, so it
 * works on seq_strict and sharded handles alike; only a handle inside a stepping call is refused. Same error
 * convention as kaminpar_b200_lp.h (0 = ok, kmp_last_error()). No CPU fallback: every call fails without a GPU.
 */
#ifndef KAMINPAR_B200_VALIDATE_H
#define KAMINPAR_B200_VALIDATE_H

#include <stddef.h>
#include <stdint.h>

#include "kaminpar_b200_lp.h"

#ifdef __cplusplus
extern "C" {
#endif

enum {
  KMP_GRAPH_VALID = 0,
  KMP_GRAPH_XADJ_START = 1,                          /* e = xadj[0] */
  KMP_GRAPH_XADJ_END = 2,                            /* u = n, e = xadj[n] */
  KMP_GRAPH_XADJ_DECREASING = 3,                     /* u */
  KMP_GRAPH_NEIGHBOR_OUT_OF_GRAPH = 4,               /* u, e, v */
  KMP_GRAPH_SELF_LOOP = 5,                           /* u, e, v */
  KMP_GRAPH_NEIGHBOR_OF_NEIGHBOR_OUT_OF_GRAPH = 6,   /* u, e, v, e_rev = q, v_rev = adjncy[q] */
  KMP_GRAPH_MISSING_REVERSE = 7,                     /* u, e, v */
  KMP_GRAPH_WEIGHT_MISMATCH = 8,                     /* u, e, v, e_rev = p, v_rev = u, w = adjwgt[e], w_rev */
  KMP_GRAPH_NUM_KINDS = 9
};

typedef struct kmp_graph_report {
  int32_t valid; /* 1: no violation (duplicates do not count) */
  int32_t kind;  /* KMP_GRAPH_*: the first violation */
  uint32_t n, m;
  /* the first violation; fields its kind does not list above are 0 */
  uint32_t u, e, v, e_rev, v_rev;
  int32_t w, w_rev;
  /* per kind: 0 or 1 for the shape kinds, the number of vertices u with xadj[u] > xadj[u+1] for
   * XADJ_DECREASING, the number of edges whose first kind it is for the edge kinds; count[0] is 0 */
  uint32_t count[KMP_GRAPH_NUM_KINDS];
  uint32_t duplicates;   /* edges whose target appeared earlier in the same row */
  uint32_t dup_u, dup_e; /* the first duplicate (both 0 without one) */
  float device_ms;       /* whole call on the device (H2D of a host input excluded) */
} kmp_graph_report;

/* Validates host arrays (copied to the device first). KMP_OK whenever the check ran, valid or not: the verdict is in
 * *out. Refused: a NULL h / out / xadj, or adjncy NULL with m > 0: KMP_ERR_INVALID; n or m >= 2^31:
 * KMP_ERR_UNSUPPORTED; not enough device memory for the copies and the scratch: KMP_ERR_ALLOC, before any kernel
 * runs; a handle inside a stepping call: KMP_ERR_INVALID. adjwgt NULL: unit edge weights (no weight check). */
int kmp_validate_graph(kmp_lp_handle *h, uint32_t n, uint32_t m, const uint32_t *xadj, const uint32_t *adjncy,
                       const int32_t *adjwgt, kmp_graph_report *out);
/* The same from device arrays on h's device; they must be 4-byte aligned (else KMP_ERR_INVALID) and are only read. */
int kmp_validate_graph_device(kmp_lp_handle *h, uint32_t n, uint32_t m, const uint32_t *d_xadj,
                              const uint32_t *d_adjncy, const int32_t *d_adjwgt, kmp_graph_report *out);

/* The reference's LOG_WARNING line for the report's first violation (without colour, "[Warning] " and newline; ""
 * for a valid report), NUL-terminated into buf[size] (truncated to fit). Returns the full length, as snprintf does.
 * Pure host code. */
int kmp_graph_report_message(const kmp_graph_report *r, char *buf, size_t size);

#ifdef __cplusplus
}
#endif
#endif
