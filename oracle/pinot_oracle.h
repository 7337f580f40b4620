/*
 * pinot_oracle.h — CPU restatement of Apache Pinot's per-segment
 * filter -> project -> group-by/aggregate path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product path (pinot_b200/, the
 * C-ABI library) may include, link or call this.  Only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs use it.
 *
 * Parity status: PINNED against the reference's own golden values
 * (pinot-core/src/test/java/org/apache/pinot/queries/
 *  InnerSegmentAggregationSingleValueQueriesTest.java:43-177 incl. the filtered aggregations :62-93,
 *  InterSegmentAggregationSingleValueQueriesTest.java:47-258,
 *  InterSegmentGroupBySingleValueQueriesTest.java:61-288) through
 * tests/test_oracle_golden.py over tests/golden/test_data_sv.npz (derived from
 * the reference's test_data-sv.avro by tests/golden/make_golden.py).
 * RoaringBitmap byte-format parity is UNPINNED (no golden bytes exist in the
 * reference; the format follows the public portable-format spec).
 *
 * CTR  = pinot-core/src/main/java/org/apache/pinot/core
 * SEGL = pinot-segment-local/src/main/java/org/apache/pinot/segment/local
 */
#ifndef PINOT_ORACLE_H
#define PINOT_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { ORC_INT = 0, ORC_LONG = 1, ORC_FLOAT = 2, ORC_DOUBLE = 3, ORC_STRING = 4 };
enum { ORC_EQ = 0, ORC_NEQ = 1, ORC_IN = 2, ORC_NOT_IN = 3, ORC_RANGE = 4, ORC_IS_NULL = 5, ORC_IS_NOT_NULL = 6 };
enum { ORC_AND = 0, ORC_OR = 1, ORC_NOT = 2, ORC_PRED = 3 };
enum { ORC_COUNT = 0, ORC_SUM = 1, ORC_MIN = 2, ORC_MAX = 3, ORC_AVG = 4, ORC_DISTINCTCOUNT = 5 };

typedef struct orc_column {
  int32_t data_type;
  int32_t has_dictionary;
  int32_t is_sorted;
  int32_t cardinality;
  int32_t bits_per_element;
  int32_t dict_entry_bytes;
  const uint8_t* forward_index;  int64_t forward_index_len;
  const uint8_t* dictionary;     int64_t dictionary_len;
  const uint8_t* inverted_index; int64_t inverted_index_len;   /* NULL when absent */
  const uint8_t* null_value_vector; int64_t null_value_vector_len;   /* .bitmap.nullvalue: RoaringBitmap of the null docIds, NULL when absent */
} orc_column;

typedef struct orc_segment {
  int32_t num_docs;
  int32_t num_columns;
  const orc_column* columns;
} orc_segment;

/* A predicate with its literal(s); lowering to dictIds happens inside the oracle. */
typedef struct orc_predicate {
  int32_t type;               /* ORC_EQ .. ORC_RANGE */
  int32_t column;             /* index into orc_segment.columns */
  int32_t num_values;         /* EQ/NEQ: 1, IN/NOT_IN: n, RANGE: 2 = {lower, upper} */
  int32_t lower_unbounded, upper_unbounded, lower_inclusive, upper_inclusive;  /* RANGE */
  int32_t _pad;
  const int64_t* int_values;  /* INT / LONG columns */
  const double* double_values;/* FLOAT / DOUBLE columns */
  const char* const* string_values;   /* STRING columns, NUL-terminated */
} orc_predicate;

/* Filter tree in postfix order. */
typedef struct orc_filter_node {
  int32_t kind;          /* ORC_AND / ORC_OR (n_children operands), ORC_NOT (1), ORC_PRED */
  int32_t n_children;
  int32_t predicate;     /* index into predicates for ORC_PRED */
} orc_filter_node;

/* A filter of its own: the FILTER(WHERE ...) clause of one or more aggregations. */
typedef struct orc_filter_program {
  int32_t num_nodes;
  int32_t _pad;
  const orc_filter_node* nodes;
  const orc_predicate* predicates;
} orc_filter_program;

typedef struct orc_aggregation {
  int32_t op;            /* ORC_COUNT .. ORC_DISTINCTCOUNT */
  int32_t column;        /* -1 for COUNT(*) */
} orc_aggregation;

typedef struct orc_query {
  int32_t num_filter_nodes;              /* 0 => match all */
  int32_t num_group_by;                  /* 0 => AggregationOperator */
  int32_t num_aggregations;
  int32_t num_groups_limit;              /* InstancePlanMakerImplV2 default 100000 */
  int32_t max_initial_result_holder_capacity;   /* default 10000 */
  int32_t skip_inverted_index;           /* query option skipIndexes: no inverted index on any column */
  const orc_filter_node* filter_nodes;
  const orc_predicate* predicates;
  const int32_t* group_by_columns;
  const orc_aggregation* aggregations;
  /* filtered aggregations (FilteredGroupByOperator / FilteredAggregationOperator): distinct FILTER clauses and, per
   * aggregation, the index of its clause (-1 = not filtered).  num_agg_filters = 0: the plain operators. */
  int32_t num_agg_filters;
  int32_t null_handling;                 /* query option enableNullHandling (QueryContext.isNullHandlingEnabled) */
  const orc_filter_program* agg_filters;
  const int32_t* agg_filter_of;
} orc_query;

typedef struct orc_stats {
  int64_t num_docs_scanned;
  int64_t num_entries_scanned_in_filter;
  int64_t num_entries_scanned_post_filter;
  int64_t num_total_docs;
  int32_t num_groups_limit_reached;
  int32_t key_holder;        /* 0 keyless, 1 ARRAY, 2 INT_MAP, 3 LONG_MAP, 4 ARRAY_MAP, 5 NO_DICT */
} orc_stats;

typedef struct orc_result orc_result;

/* Run GroupByOperator / AggregationOperator over one segment.  Returns NULL on
 * error (orc_last_error()). */
orc_result* orc_execute(const orc_segment* seg, const orc_query* q);
void orc_result_free(orc_result* r);
const char* orc_last_error(void);
/* the segments of one query on `threads` worker threads (shared work queue); out[i] = result of segment i; returns the number
 * of segments that failed */
int32_t orc_execute_batch(const orc_segment* const* segs, const orc_query* const* qs, int32_t n, int32_t threads, orc_result** out);
/* the same pass with the cross-segment merge (GroupByCombineOperator / IndexedTable) done natively by the worker threads */
int64_t orc_execute_combined(const orc_segment* const* segs, const orc_query* const* qs, int32_t n, int32_t threads,
                             int64_t** keys_out, double** dbl_out, int64_t** lng_out);

int32_t orc_result_num_groups(const orc_result* r);        /* 1 for keyless */
const orc_stats* orc_result_stats(const orc_result* r);
/* group keys [num_groups][num_group_by]: the dictId for a dictionary column, the raw value bits
 * (sign-extended INT / LONG, IEEE bits of the double for FLOAT / DOUBLE) for a raw column. */
const int64_t* orc_result_group_keys(const orc_result* r);
/* per aggregation arrays of length num_groups */
const double* orc_result_double(const orc_result* r, int32_t agg);   /* SUM, MIN, MAX, AVG sum */
const int64_t* orc_result_long(const orc_result* r, int32_t agg);    /* COUNT, AVG count, DISTINCTCOUNT size */
/* DISTINCTCOUNT value sets: offsets[num_groups+1] into ids[] (dictIds, ascending per group) */
const int64_t* orc_result_distinct_offsets(const orc_result* r, int32_t agg);
const int32_t* orc_result_distinct_dict_ids(const orc_result* r, int32_t agg);
/* DISTINCTCOUNT on a raw column: the value sets as bits (INT / LONG: the value; FLOAT / DOUBLE: IEEE bits of the double), NULL otherwise */
const int64_t* orc_result_distinct_values(const orc_result* r, int32_t agg);

/* Matching docIds of the filter alone (ascending, as DocIdSetOperator would deliver them);
 * returns the count, *out is malloc'd (orc_free). */
int64_t orc_filter_doc_ids(const orc_segment* seg, const orc_query* q, int32_t** out, int64_t* entries_scanned);
void orc_free(void* p);

/* small helpers exposed for unit tests */
int32_t orc_num_bits_per_value(int32_t max_value);
int32_t orc_read_dict_id(const uint8_t* fwd, int32_t bits, int64_t doc);
int64_t orc_roaring_to_doc_ids(const uint8_t* blob, int64_t len, uint32_t* out, int64_t cap);
/* chunk codecs of raw forward indexes (LZ4 block / raw Snappy) and the whole-index rewrite to PASS_THROUGH */
int64_t orc_lz4_block_decode(const uint8_t* in, int64_t in_len, uint8_t* out, int64_t out_cap);
int64_t orc_snappy_block_decode(const uint8_t* in, int64_t in_len, uint8_t* out, int64_t out_cap);
int64_t orc_raw_forward_decompress(const uint8_t* fwd, int64_t len, int32_t width, int32_t num_docs, uint8_t* out, int64_t out_cap);

#ifdef __cplusplus
}
#endif
#endif
