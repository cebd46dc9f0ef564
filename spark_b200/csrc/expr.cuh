// expr.cuh -- FilterExec / ProjectExec expression programs (sb_expr) on the GPU.
#pragma once
#include "common.cuh"

namespace sb {

constexpr int EXPR_MAX_NODES = 48;
constexpr int EXPR_STACK = 12;

// validates the program against the table (column indices/types, stack discipline) -- host only
void expr_validate(const sb_table *in, const sb_expr &e);
// true if the expression is a bare column reference (ProjectExec of an attribute)
bool expr_is_column(const sb_expr &e, int *col);
// can the result contain NULLs?
bool expr_nullable(const sb_table *in, const sb_expr &e);

// mask[i] = 1 when the predicate is TRUE (not NULL) for row i; validates the program first (also for an empty table)
void eval_predicate(const sb_table *in, const sb_expr &pred, uint8_t *mask_dev, cudaStream_t st);
// materialises the expression for rows sel[0..nout) (sel == nullptr -> rows 0..nout); validates it unless it is a bare column
Column eval_projection(const sb_table *in, const sb_expr &e, const int64_t *sel, int64_t nout, cudaStream_t st);

}  // namespace sb
