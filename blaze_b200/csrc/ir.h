// Host-side plan IR of the hot path: what plan decoding (auron-serde/src/from_proto.rs:107-152,
// 407-500, 839-1026) produces, restricted to Filter / Projection / Agg over fixed-width columns.
#pragma once
#include <cstdint>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

namespace b200q {

// must match blaze_b200/types.py
enum TypeId : uint8_t { T_BOOL = 0, T_INT8, T_INT16, T_INT32, T_INT64, T_FLOAT32, T_FLOAT64, T_DATE32,
                        T_TIMESTAMP_US, T_DECIMAL128, T_BINARY, T_NULL, T_UTF8 };

struct DType {
  TypeId id = T_NULL;
  uint8_t precision = 0;
  int8_t scale = 0;
  bool operator==(const DType& o) const { return id == o.id && precision == o.precision && scale == o.scale; }
  bool operator!=(const DType& o) const { return !(*this == o); }
  bool is_integer() const { return id >= T_INT8 && id <= T_INT64; }
  bool is_float() const { return id == T_FLOAT32 || id == T_FLOAT64; }
  bool is_decimal() const { return id == T_DECIMAL128; }
  // offsets + data buffers (Arrow Utf8 / Binary): imported, exported and carried through one code path
  bool is_varlen() const { return id == T_UTF8 || id == T_BINARY; }
  // ints, bool, date32, timestamp all travel as sign-extended i64 on the device
  bool is_intlike() const { return is_integer() || id == T_BOOL || id == T_DATE32 || id == T_TIMESTAMP_US; }
  int byte_width() const {
    switch (id) {
      case T_BOOL: return 0;  // bit-packed
      case T_INT8: return 1; case T_INT16: return 2; case T_INT32: case T_FLOAT32: case T_DATE32: return 4;
      case T_INT64: case T_FLOAT64: case T_TIMESTAMP_US: return 8; case T_DECIMAL128: return 16;
      default: return 0;
    }
  }
  int int_bits() const {
    switch (id) { case T_BOOL: return 1; case T_INT8: return 8; case T_INT16: return 16; case T_INT32: case T_DATE32: return 32; default: return 64; }
  }
  std::string str() const;
};

struct FieldDef { std::string name; DType type; bool nullable = true; };
struct SchemaDef {
  std::vector<FieldDef> fields;
  int index_of(const std::string& name) const {
    for (size_t i = 0; i < fields.size(); i++) if (fields[i].name == name) return (int)i;
    return -1;
  }
};

struct PlanError : std::runtime_error {
  int code;
  PlanError(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

enum ExprKind : uint8_t { E_COLUMN, E_LITERAL, E_BINARY, E_IS_NULL, E_IS_NOT_NULL, E_NOT, E_NEGATIVE, E_CAST,
                          E_TRY_CAST, E_CASE, E_IN_LIST, E_SC_AND, E_SC_OR, E_SCALAR_FN, E_STR_MATCH };
// E_STR_MATCH: StringStartsWith / EndsWith / Contains ExprNode (auron.proto:339-352); pattern in lit_str
enum StrMatch : uint8_t { SM_STARTS_WITH = 0, SM_ENDS_WITH, SM_CONTAINS };
enum BinOp : uint8_t { OP_AND, OP_OR, OP_EQ, OP_NE, OP_LT, OP_LE, OP_GT, OP_GE, OP_PLUS, OP_MINUS, OP_MUL, OP_DIV,
                       OP_MOD, OP_BIT_AND, OP_BIT_OR, OP_BIT_XOR };

struct Expr;
using ExprP = std::shared_ptr<Expr>;

struct Expr {
  ExprKind kind;
  DType type;             // result type (inferred at decode time)
  bool nullable = true;   // DataFusion PhysicalExpr::nullable
  // E_COLUMN
  int col_index = -1;
  std::string name;       // column name / scalar function name
  // E_LITERAL: value bits (decimal: lo/hi of the i128; float: IEEE bits of f64 (f32 widened); int: sign-extended)
  bool lit_null = false;
  uint64_t lit_lo = 0, lit_hi = 0;
  std::string lit_str;    // Utf8 literal bytes; also the pattern of E_STR_MATCH
  // E_BINARY
  BinOp op = OP_AND;
  // E_IN_LIST
  bool negated = false;
  // E_STR_MATCH
  StrMatch str_match = SM_STARTS_WITH;
  // E_CASE: children = [base?] w1 t1 w2 t2 ... [else]; flags say which are present
  bool case_has_base = false, case_has_else = false;
  std::vector<ExprP> children;
};

enum AggFn : uint8_t { AGG_MIN = 0, AGG_MAX = 1, AGG_SUM = 2, AGG_AVG = 3, AGG_COUNT = 4 };
enum AggMode : uint8_t { MODE_PARTIAL = 0, MODE_PARTIAL_MERGE = 1, MODE_FINAL = 2 };

struct AggDef {
  AggFn fn;
  AggMode mode;
  std::string field_name;
  DType data_type;              // Agg::data_type(): Sum/Avg = return_type, Min/Max = child type, Count = Int64
  std::vector<ExprP> args;      // after create_agg rewriting: Sum/Avg -> TryCast(child,rt); Count -> nullable children only
  bool nullable() const { return fn != AGG_COUNT; }
  DType final_type() const {    // type of the Final-mode output column
    if (fn == AGG_AVG && !data_type.is_decimal()) { DType d; d.id = T_FLOAT64; return d; }
    return data_type;
  }
};

enum NodeKind : uint8_t { N_LEAF, N_FILTER, N_PROJECT, N_AGG, N_SHUFFLE_WRITER, N_JOIN_BUILD, N_JOIN, N_SORT, N_EXPAND, N_WINDOW };
enum ShuffleKind : uint8_t { SHUFFLE_SINGLE = 0, SHUFFLE_HASH = 1, SHUFFLE_ROUND_ROBIN = 2, SHUFFLE_RANGE = 3 };   // PhysicalRepartition oneof (auron.proto:629-655)

struct PlanNode {
  NodeKind kind;
  SchemaDef schema;                        // output schema of this node
  std::shared_ptr<PlanNode> input;
  // N_LEAF
  std::string leaf_kind;                   // "FFIReader" | "EmptyPartitions"
  std::string resource_id;
  // N_FILTER
  std::vector<ExprP> predicates;
  // N_PROJECT
  std::vector<ExprP> proj_exprs;           // already wrapped in TryCast when the declared type differs
  // N_AGG
  int exec_mode = 0;
  std::vector<ExprP> group_exprs;
  std::vector<std::string> group_names;
  std::vector<AggDef> aggs;
  bool supports_partial_skipping = false;
  bool need_final_merge = false, need_partial_update = false, need_partial_merge = false;
  // N_SHUFFLE_WRITER (ShuffleWriterExecNode, auron.proto:524-529)
  ShuffleKind shuffle_kind = SHUFFLE_SINGLE;
  uint64_t num_partitions = 1;
  std::vector<ExprP> hash_exprs;
  std::string data_file, index_file;
  // N_JOIN_BUILD (BroadcastJoinBuildHashMapExecNode, auron.proto:450-453): keys resolved against the input schema
  std::vector<ExprP> join_build_keys;
  // N_JOIN (HashJoinExecNode / BroadcastJoinExecNode, auron.proto:441-463): `input` is the PROBED child, `join_build`
  // the child whose rows are in the hash map (its subtree only supplies the schema: the map comes from a build op)
  std::shared_ptr<PlanNode> join_build;
  bool join_build_is_left = false;
  int join_type = 0;                                                  // protobuf JoinType (auron.proto:475-483)
  std::vector<std::pair<ExprP, ExprP>> join_on;                       // (left key, right key)
  SchemaDef join_left_schema, join_right_schema;
  std::string cached_build_hash_map_id;
  // N_LEAF, leaf_kind "ParquetScan" (ParquetScanExecNode + FileScanExecConf, auron.proto:368-419)
  struct ScanFile { std::string path; uint64_t size = 0; bool has_range = false; int64_t range_start = 0, range_end = 0; };
  std::vector<ScanFile> scan_files;
  SchemaDef scan_file_schema;                                         // base_conf.schema: the file's columns as Spark sees them
  std::vector<int> scan_projection;                                   // indices into scan_file_schema (empty: every column)
  std::vector<ExprP> scan_pruning;                                    // pruning_predicates, resolved against scan_file_schema
  bool scan_has_limit = false; uint64_t scan_limit = 0;
  // N_SORT (SortExecNode, auron.proto:618-627; PhysicalSortExprNode :178-182)
  struct SortExprDef { ExprP expr; bool asc = true; bool nulls_first = true; };
  std::vector<SortExprDef> sort_exprs;
  bool sort_has_fetch = false;
  uint64_t sort_fetch = 0;
  // N_EXPAND (ExpandExecNode, auron.proto:714-722): one expression per schema field in every projection, resolved against
  // the input schema, of exactly the field's type (expressions beyond the field count are dropped at decode)
  std::vector<std::vector<ExprP>> expand_projections;
  // N_WINDOW (WindowExecNode / WindowExprNode, auron.proto:537-562): expressions resolved against the input schema.  Output =
  // input columns ++ (output_window_cols ? one column per window expression : nothing)
  struct WindowExprDef {
    FieldDef field;
    bool is_rank = true;
    int rank_fn = 0;                       // WindowFunction: 0 ROW_NUMBER, 1 RANK, 2 DENSE_RANK
    AggDef agg;                            // is_rank false: args after create_agg rewriting (as AggExec), mode Partial
  };
  std::vector<WindowExprDef> window_exprs;
  std::vector<ExprP> window_partition;
  std::vector<SortExprDef> window_order;
  bool window_has_limit = false;
  uint32_t window_limit = 0;
  bool output_window_cols = false;
};
using PlanP = std::shared_ptr<PlanNode>;

// WindowExec limits, refused at decode (UNSUPPORTED)
constexpr int WINDOW_MAX_EXPRS = 8;        // window expressions of one node
constexpr int WINDOW_MAX_KEYS = 16;        // partition + order keys
constexpr int WINDOW_MAX_COUNT_ARGS = 4;   // nullable COUNT arguments

// plan_decode.cc
PlanP decode_plan(const uint8_t* bytes, size_t n, int plan_kind);
std::string explain_plan(const PlanP& p);
std::string explain_expr(const ExprP& e);
constexpr const char* AGG_BUF_COLUMN_NAME = "#9223372036854775807";   // agg/mod.rs:37

// arrow_ipc.cc: ScalarValue.ipc_bytes -> literal Expr (auron-serde/src/lib.rs:447-457)
ExprP decode_ipc_literal(const uint8_t* bytes, size_t n);

}  // namespace b200q
