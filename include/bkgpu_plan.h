/*
 * bkgpu_plan.h — POD mirror of the reference's plan / expression description.
 *
 * The reference ships plan fragments as protobuf (`pb::Plan`, `pb::Expr`;
 * /root/reference/proto/plan.proto:495-511, proto/expr.proto:67-84) and rebuilds
 * the operator / expression trees from their PRE-ORDER node lists
 * (src/exec/exec_node.cpp:361-394, src/expr/expr_node.cpp:415-445).  The C ABI
 * in bkgpu.h takes the same information as a flat little-endian stream of
 * 32-bit words so that no protobuf type crosses the boundary.  Enum VALUES are
 * the reference's own (a maintainer's adapter copies them straight out of the
 * pb objects); only the container is new.
 *
 * Stream grammar (every token is one int32 word unless marked 64 = two words,
 * low word first; STR = length word + bytes zero-padded to a multiple of 4):
 *
 *   PLAN  := MAGIC VERSION n_tuples n_nodes TUPLE* NODE*            (NODE* pre-order)
 *   TUPLE := tuple_id n_slots (slot_id prim_type)*                   pb::TupleDescriptor
 *   NODE  := node_type num_children limit64 PAYLOAD                  pb::PlanNode
 *     SCAN_NODE                      : tuple_id table_id64
 *     WHERE/TABLE/HAVING_FILTER_NODE : n_conjuncts EXPR*             pb::FilterNode.conjuncts
 *     AGG_NODE / MERGE_AGG_NODE      : agg_tuple_id n_group EXPR* n_agg EXPR*   pb::AggNode
 *     SORT_NODE                      : tuple_id n_order (EXPR is_asc is_null_first)*  pb::SortNode
 *     JOIN_NODE                      : join_type n_conditions EXPR*  pb::JoinNode
 *     APPLY_NODE                     : join_type n_conditions EXPR* max_one_row compare_type is_select_field   pb::ApplyNode
 *                                      (child 0 = outer query, child 1 = subquery; their scan tuples are the outer / inner tuples, so
 *                                       left / right tuple id lists are not carried.  compare_type: CMP_NULL 0, ANY 1, ALL 2, SOME 3)
 *     LIMIT_NODE                     : offset64                      pb::LimitNode
 *     WINDOW_NODE                    : n_fn EXPR* n_part EXPR* n_order (EXPR is_asc)* has_frame [FRAME]   pb::WindowNode
 *       FRAME := frame_type BOUND(start) BOUND(end)                  pb::WindowFrame (FT_ROWS 0, FT_RANGE 1)
 *       BOUND := bound_type is_unbounded has_expr [EXPR]             pb::FrameBound (BT_PRECEDING 0, BT_FOLLOWING 1, BT_CURRENT_ROW 2)
 *     PACKET_NODE / SELECT_MANAGER_NODE : (nothing; accepted and skipped)
 *   EXPR  := n_nodes ENODE*                                          (ENODE* pre-order)
 *   ENODE := node_type col_type num_children PAYLOAD                 pb::ExprNode
 *     SLOT_REF        : tuple_id slot_id
 *     NULL_LITERAL    : -
 *     BOOL_LITERAL    : value
 *     INT_LITERAL     : value64
 *     DOUBLE_LITERAL  : ieee754-bits64
 *     STRING_LITERAL  : str (taken only where it meets a DATE / DATETIME / TIMESTAMP / TIME operand: folded into that type's image
 *                       the way ExprValue::cast_to parses it, include/common/expr_value.h:534-573)
 *     DATETIME_LITERAL, TIMESTAMP_LITERAL, DATE_LITERAL, TIME_LITERAL : value64 = the image (DeriveExprNode.int_val, literal.h:95-114)
 *     FUNCTION_CALL, *_PREDICATE : fn_op STR(name) n_arg_types arg_type* return_type   pb::Function
 *                       (n_arg_types == 0 / return_type == 0: not yet completed; the library
 *                        then runs the reference's type inference itself —
 *                        ScalarFnCall::type_inferer + FunctionManager::complete_fn,
 *                        src/expr/scalar_fn_call.cpp:40-120, src/expr/fn_manager.cpp:316-409)
 *     AGG_EXPR        : STR(name) tuple_id final_slot_id intermediate_slot_id
 *     WINDOW_EXPR     : STR(name) tuple_id slot_id                   pb::Function.name + DeriveExprNode (window_fn_call.cpp:19-63)
 */
#ifndef BKGPU_PLAN_H_
#define BKGPU_PLAN_H_

#include <stdint.h>

#define BKGPU_PLAN_MAGIC   0x31504B42u /* "BKP1" */
#define BKGPU_PLAN_VERSION 1

/* pb::PlanNodeType — proto/plan.proto:9-53 */
enum bkgpu_plan_node_type {
    BK_SCAN_NODE = 1, BK_SORT_NODE = 2, BK_AGG_NODE = 4, BK_MERGE_AGG_NODE = 5,
    BK_TABLE_FILTER_NODE = 6, BK_JOIN_NODE = 7, BK_LIMIT_NODE = 11,
    BK_WHERE_FILTER_NODE = 12, BK_HAVING_FILTER_NODE = 13, BK_PACKET_NODE = 14,
    BK_SELECT_MANAGER_NODE = 25, BK_APPLY_NODE = 37, BK_WINDOW_NODE = 42
};

/* pb::ExprNodeType — proto/expr.proto:6-37 */
enum bkgpu_expr_node_type {
    BK_SLOT_REF = 1, BK_FUNCTION_CALL = 2, BK_AGG_EXPR = 3, BK_NULL_LITERAL = 4,
    BK_BOOL_LITERAL = 5, BK_INT_LITERAL = 6, BK_DOUBLE_LITERAL = 7, BK_STRING_LITERAL = 8,
    BK_IS_NULL_PREDICATE = 9, BK_IN_PREDICATE = 10, BK_LIKE_PREDICATE = 11,
    BK_NOT_PREDICATE = 12, BK_AND_PREDICATE = 13, BK_OR_PREDICATE = 14,
    BK_XOR_PREDICATE = 15, BK_TIMESTAMP_LITERAL = 16, BK_DATETIME_LITERAL = 17, BK_DATE_LITERAL = 18,
    BK_IS_TRUE_PREDICATE = 19, BK_TIME_LITERAL = 20, BK_ROW_EXPR = 22, BK_WINDOW_EXPR = 30
};

/* pb::FrameType / pb::BoundType — proto/plan.proto:427-436 */
enum bkgpu_frame_type { BK_FRAME_ROWS = 0, BK_FRAME_RANGE = 1 };
enum bkgpu_bound_type { BK_BT_PRECEDING = 0, BK_BT_FOLLOWING = 1, BK_BT_CURRENT_ROW = 2 };

/* pb::PrimitiveType — proto/common.proto:46-72 */
enum bkgpu_primitive_type {
    BK_INVALID_TYPE = 0, BK_NULL_TYPE = 1, BK_BOOL = 2, BK_INT8 = 3, BK_INT16 = 4,
    BK_INT32 = 5, BK_INT64 = 6, BK_UINT8 = 7, BK_UINT16 = 8, BK_UINT32 = 9,
    BK_UINT64 = 10, BK_FLOAT = 11, BK_DOUBLE = 12, BK_STRING = 13, BK_DATETIME = 14,
    BK_TIMESTAMP = 15, BK_DATE = 16, BK_HLL = 17, BK_TIME = 18, BK_BITMAP = 21
};

/* parser::FuncType carried in pb::Function.fn_op — include/sqlparser/expr.h:48-89 */
enum bkgpu_func_type {
    BK_FT_COMMON = 0, BK_FT_AGG = 1, BK_FT_BIT_NOT = 2, BK_FT_LOGIC_NOT = 3, BK_FT_UMINUS = 4,
    BK_FT_ADD = 5, BK_FT_MINUS = 6, BK_FT_MULTIPLIES = 7, BK_FT_DIVIDES = 8, BK_FT_MOD = 9,
    BK_FT_LS = 10, BK_FT_RS = 11, BK_FT_BIT_AND = 12, BK_FT_BIT_OR = 13, BK_FT_BIT_XOR = 14,
    BK_FT_EQ = 15, BK_FT_NE = 16, BK_FT_GT = 17, BK_FT_GE = 18, BK_FT_LT = 19, BK_FT_LE = 20,
    BK_FT_LOGIC_AND = 21, BK_FT_LOGIC_OR = 22, BK_FT_LOGIC_XOR = 23, BK_FT_IS_NULL = 24,
    BK_FT_IS_TRUE = 25, BK_FT_IS_UNKNOWN = 26, BK_FT_IN = 27, BK_FT_LIKE = 28
};

/* pb::JoinType — proto/plan.proto:218-226 */
enum bkgpu_join_type {
    BK_NULL_JOIN = 0, BK_LEFT_JOIN = 1, BK_RIGHT_JOIN = 2, BK_INNER_JOIN = 3,
    BK_SEMI_JOIN = 4, BK_ANTI_SEMI_JOIN = 5, BK_FULL_JOIN = 6
};

/* pb::CompareType — proto/plan.proto:239-244 (ApplyNode.compare_type) */
enum bkgpu_compare_type { BK_CMP_NULL = 0, BK_CMP_ANY = 1, BK_CMP_ALL = 2, BK_CMP_SOME = 3 };

#endif /* BKGPU_PLAN_H_ */
