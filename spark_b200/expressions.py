"""Catalyst-style expression nodes for the GPU operators.

Names and semantics mirror sql/catalyst/src/main/scala/org/apache/spark/sql/catalyst/expressions of the
reference (arithmetic.scala, predicates.scala, nullExpressions.scala, Cast.scala, aggregate/*.scala); only the
subset the shuffle / sort / aggregate / join path needs.  `compile()` lowers a tree to the postfix sb_expr
program of include/spark_b200.h; `sexpr()` gives the neutral nested-tuple form the test oracle consumes.
"""
from __future__ import annotations

import ctypes as C
import datetime
import struct

from . import _capi as capi

VT_BOOL, VT_I32, VT_I64, VT_F64 = capi.SB_VT_BOOL, capi.SB_VT_I32, capi.SB_VT_I64, capi.SB_VT_F64

_VT_OF_SB = {capi.SB_BOOL: VT_BOOL, capi.SB_INT8: VT_I32, capi.SB_INT16: VT_I32, capi.SB_INT32: VT_I32,
             capi.SB_DATE32: VT_I32, capi.SB_INT64: VT_I64, capi.SB_TIMESTAMP: VT_I64, capi.SB_DECIMAL64: VT_I64,
             capi.SB_FLOAT32: VT_F64, capi.SB_FLOAT64: VT_F64}
_OUT_OF_VT = {VT_BOOL: capi.SB_BOOL, VT_I32: capi.SB_INT32, VT_I64: capi.SB_INT64, VT_F64: capi.SB_FLOAT64}


class Schema:
    """names + physical sb types of an operator's input (the `output: Seq[Attribute]` of a SparkPlan)."""

    def __init__(self, names, types, binary=()):
        self.names = list(names)
        self.types = list(types)
        self.binary = set(binary)        # SB_STRING columns whose values are binary, not strings (Length counts their bytes)

    def index(self, name):
        try:
            return self.names.index(name)
        except ValueError:
            raise KeyError("unresolved attribute %r among %r" % (name, self.names))


class Expression:
    children = ()

    def vtype(self, schema) -> int:
        raise NotImplementedError

    def emit(self, schema, out):
        raise NotImplementedError

    def sexpr(self):
        raise NotImplementedError

    def references(self):
        r = set()
        for c in self.children:
            r |= c.references()
        return r

    # operator sugar
    def __add__(self, o): return Add(self, _wrap(o))
    def __radd__(self, o): return Add(_wrap(o), self)
    def __sub__(self, o): return Subtract(self, _wrap(o))
    def __rsub__(self, o): return Subtract(_wrap(o), self)
    def __mul__(self, o): return Multiply(self, _wrap(o))
    def __rmul__(self, o): return Multiply(_wrap(o), self)
    def __truediv__(self, o): return Divide(self, _wrap(o))
    def __neg__(self): return UnaryMinus(self)
    def __lt__(self, o): return LessThan(self, _wrap(o))
    def __le__(self, o): return LessThanOrEqual(self, _wrap(o))
    def __gt__(self, o): return GreaterThan(self, _wrap(o))
    def __ge__(self, o): return GreaterThanOrEqual(self, _wrap(o))
    def eq(self, o): return EqualTo(self, _wrap(o))
    def ne(self, o): return Not(EqualTo(self, _wrap(o)))
    def __and__(self, o): return And(self, _wrap(o))
    def __or__(self, o): return Or(self, _wrap(o))
    def __invert__(self): return Not(self)
    def is_null(self): return IsNull(self)
    def is_not_null(self): return IsNotNull(self)


def _wrap(x):
    return x if isinstance(x, Expression) else Literal(x)


def _node(op, vtype, arg=0, lit_i=None, lit_d=None, arg2=0):
    n = capi.sb_expr_node()
    n.op = capi.SB_OP[op]
    n.vtype = vtype
    n.arg = arg
    n.arg2 = arg2
    if lit_d is not None:
        n.lit.d = lit_d
    elif lit_i is not None:
        n.lit.i = lit_i
    return n


class AttributeReference(Expression):
    def __init__(self, name):
        self.name = name

    def vtype(self, schema):
        t = schema.types[schema.index(self.name)]
        # strings and decimal(p > 18) have no value class: they are only moved as bare references (the native side refuses them
        # in arithmetic or comparisons).  Filter and expand over a decimal(38, s) column used to stop here with a KeyError
        # (caught by test_gpu_row_movement.py::test_filter / test_expand).
        if t in (capi.SB_STRING, capi.SB_DECIMAL128):
            return 0
        return _VT_OF_SB[t]

    def emit(self, schema, out):
        out.append(_node("COL", self.vtype(schema), schema.index(self.name)))

    def sexpr(self):
        return ("col", self.name)

    def references(self):
        return {self.name}


col = AttributeReference


class Literal(Expression):
    def __init__(self, value, vt=None):
        if isinstance(value, datetime.date):
            value = (value - datetime.date(1970, 1, 1)).days
            vt = vt or VT_I32
        self.value = value
        if vt is None:
            if isinstance(value, (str, bytes)):
                vt = 0                       # a string: only the string tests below take one
            elif value is None:
                vt = VT_I64
            elif isinstance(value, bool):
                vt = VT_BOOL
            elif isinstance(value, float):
                vt = VT_F64
            else:
                vt = VT_I32 if -2 ** 31 <= value < 2 ** 31 else VT_I64
        self.vt = vt

    def vtype(self, schema):
        return self.vt

    def emit(self, schema, out):
        if self.vt == 0:
            raise TypeError("a string literal is only an operand of a string test (comparison, IN, LIKE, StartsWith ...)")
        if self.value is None:
            out.append(_node("LIT_NULL", self.vt))
        elif self.vt == VT_F64:
            out.append(_node("LIT_F64", VT_F64, lit_d=float(self.value)))
        else:
            out.append(_node("LIT_I64", self.vt, lit_i=int(self.value)))

    def sexpr(self):
        import numpy as np
        if self.vt == 0:
            return ("lit", self.value, type(self.value))
        dt = {VT_BOOL: bool, VT_I32: np.int32, VT_I64: np.int64, VT_F64: np.float64}[self.vt]
        return ("lit", self.value, dt)


lit = Literal


def _promote(a, b):
    """Binary numeric promotion (TypeCoercion): int32 < int64 < double."""
    return max(a, b)


class _Cast(Expression):
    def __init__(self, child, to_vt):
        self.child = child
        self.children = (child,)
        self.to = to_vt

    def vtype(self, schema):
        return self.to

    def emit(self, schema, out):
        self.child.emit(schema, out)
        src = self.child.vtype(schema)
        if src == self.to:
            return
        op = {VT_F64: "CAST_F64", VT_I64: "CAST_I64", VT_I32: "CAST_I32"}[self.to]
        out.append(_node(op, self.to, src))

    def sexpr(self):
        return ({VT_F64: "cast_f64", VT_I64: "cast_i64", VT_I32: "cast_i32"}[self.to], self.child.sexpr())


def Cast(child, to):
    vt = {"double": VT_F64, "long": VT_I64, "int": VT_I32}.get(to, to)
    return _Cast(child, vt)


def _coerce(e, schema, to_vt):
    """Implicit cast of a child to the operator's type; literals are re-typed instead of cast."""
    vt = e.vtype(schema)
    if vt == to_vt:
        return e
    if isinstance(e, Literal) and e.value is not None:
        return Literal(float(e.value) if to_vt == VT_F64 else e.value, to_vt)
    return _Cast(e, to_vt)


class _BinaryArith(Expression):
    op = None
    name = None

    def __init__(self, left, right):
        self.left, self.right = left, right
        self.children = (left, right)

    def vtype(self, schema):
        return _promote(self.left.vtype(schema), self.right.vtype(schema))

    def emit(self, schema, out):
        vt = self.vtype(schema)
        _coerce(self.left, schema, vt).emit(schema, out)
        _coerce(self.right, schema, vt).emit(schema, out)
        out.append(_node(self.op, vt))

    def sexpr(self):
        return (self.name, self.left.sexpr(), self.right.sexpr())


class Add(_BinaryArith):
    op, name = "ADD", "add"


class Subtract(_BinaryArith):
    op, name = "SUB", "sub"


class Multiply(_BinaryArith):
    op, name = "MUL", "mul"


class Divide(_BinaryArith):
    """Spark's `/` on non-decimals is double division; NULL when the divisor is 0 (non-ANSI)."""
    op, name = "DIV", "div"

    def vtype(self, schema):
        return VT_F64


class UnaryMinus(Expression):
    def __init__(self, child):
        self.child = child
        self.children = (child,)

    def vtype(self, schema):
        return self.child.vtype(schema)

    def emit(self, schema, out):
        self.child.emit(schema, out)
        out.append(_node("NEG", self.vtype(schema)))

    def sexpr(self):
        return ("neg", self.child.sexpr())


class _Comparison(Expression):
    op = None
    name = None

    def __init__(self, left, right):
        self.left, self.right = left, right
        self.children = (left, right)

    def vtype(self, schema):
        return VT_BOOL

    def _string_sides(self):
        """(column, literal bytes, flipped) when this compares a string column with a string literal, else None."""
        l, r = self.left, self.right
        if isinstance(r, (AttributeReference, StringFunction)) and _is_str_lit(l):
            return r, _utf8(l.value), True
        if isinstance(l, (AttributeReference, StringFunction)) and _is_str_lit(r):
            return l, _utf8(r.value), False
        return None

    def emit(self, schema, out):
        s = self._string_sides()
        if s is not None:                            # STR_* keeps the column on the left: 'x' < s is s > 'x'
            c, b, flipped = s
            op = _FLIP[self.op] if flipped else self.op
            out.append(_node("STR_" + op, VT_BOOL, _string_col(c, schema), lit_i=_pool(out).slice(b)))
            return
        vt = _promote(self.left.vtype(schema), self.right.vtype(schema))
        _coerce(self.left, schema, vt).emit(schema, out)
        _coerce(self.right, schema, vt).emit(schema, out)
        out.append(_node(self.op, VT_BOOL, vt))   # arg = operand class

    def sexpr(self):
        if self._string_sides() is not None:
            return ("str_cmp", self.name, self.left.sexpr(), self.right.sexpr())
        return (self.name, self.left.sexpr(), self.right.sexpr())


class EqualTo(_Comparison):
    op, name = "EQ", "eq"


class LessThan(_Comparison):
    op, name = "LT", "lt"


class LessThanOrEqual(_Comparison):
    op, name = "LE", "le"


class GreaterThan(_Comparison):
    op, name = "GT", "gt"


class GreaterThanOrEqual(_Comparison):
    op, name = "GE", "ge"


class _Logical(Expression):
    op = None
    name = None

    def __init__(self, left, right):
        self.left, self.right = left, right
        self.children = (left, right)

    def vtype(self, schema):
        return VT_BOOL

    def emit(self, schema, out):
        self.left.emit(schema, out)
        self.right.emit(schema, out)
        out.append(_node(self.op, VT_BOOL))

    def sexpr(self):
        return (self.name, self.left.sexpr(), self.right.sexpr())


class And(_Logical):
    op, name = "AND", "and"


class Or(_Logical):
    op, name = "OR", "or"


class _Unary(Expression):
    op = None
    name = None

    def __init__(self, child):
        self.child = child
        self.children = (child,)

    def vtype(self, schema):
        return VT_BOOL

    def emit(self, schema, out):
        self.child.emit(schema, out)
        out.append(_node(self.op, VT_BOOL))

    def sexpr(self):
        return (self.name, self.child.sexpr())


class Not(_Unary):
    op, name = "NOT", "not"


class IsNull(_Unary):
    op, name = "ISNULL", "isnull"


class IsNotNull(_Unary):
    op, name = "ISNOTNULL", "isnotnull"


# ---- string tests against literals (stringExpressions.scala, regexpExpressions.scala Like, predicates.scala In / InSet) --------
# Each lowers to one SB_OP_STR_* leaf naming its column; the literal bytes go to the program's pool (include/spark_b200.h).
class _Program(list):
    """The node list an expression emits into, with the pool its string literals are appended to."""

    def __init__(self):
        super().__init__()
        self.pool = bytearray()

    def slice(self, b: bytes) -> int:
        off = len(self.pool)
        self.pool += b
        return off << 32 | len(b)


def _pool(out) -> _Program:
    if not isinstance(out, _Program):
        raise TypeError("string tests are emitted through CompiledExpr")
    return out


_FLIP = {"EQ": "EQ", "LT": "GT", "LE": "GE", "GT": "LT", "GE": "LE"}


def _utf8(v) -> bytes:
    return v if isinstance(v, bytes) else v.encode("utf-8")


def _is_str_lit(e) -> bool:
    return isinstance(e, Literal) and isinstance(e.value, (str, bytes))


def _string_col(c, schema) -> int:
    if isinstance(c, StringFunction):
        raise TypeError("%s: a string function inside a numeric program is evaluated first (execution.py hoists it into a column)" % c.name)
    i = schema.index(c.name)
    if schema.types[i] != capi.SB_STRING:
        raise TypeError("%r is not a string column" % c.name)
    return i


class _StringTest(Expression):
    op = None
    name = None

    def __init__(self, child, literal):
        if not isinstance(child, (AttributeReference, StringFunction)):
            raise TypeError("string tests take a string column or a string function")
        self.child, self.literal = child, _utf8(literal)
        self.children = (child,)

    def vtype(self, schema):
        return VT_BOOL

    def emit(self, schema, out):
        out.append(_node(self.op, self.vtype(schema), _string_col(self.child, schema), lit_i=_pool(out).slice(self.literal)))

    def sexpr(self):
        return (self.name, self.child.sexpr(), self.literal)


class StartsWith(_StringTest):
    op, name = "STR_STARTS_WITH", "starts_with"


class EndsWith(_StringTest):
    op, name = "STR_ENDS_WITH", "ends_with"


class Contains(_StringTest):
    op, name = "STR_CONTAINS", "contains"


class Like(_StringTest):
    """`child LIKE pattern ESCAPE escape`: `_` one code point, `%` any run of them; the escape character may only precede `%`, `_`
    or itself (the engine refuses other patterns with SB_ERR_INVALID)."""
    op, name = "STR_LIKE", "like"

    def __init__(self, child, pattern, escape="\\"):
        super().__init__(child, pattern)
        if len(escape) != 1:
            raise ValueError("the escape must be one character")
        self.escape = escape

    def emit(self, schema, out):
        out.append(_node(self.op, VT_BOOL, _string_col(self.child, schema), lit_i=_pool(out).slice(self.literal), arg2=ord(self.escape)))

    def sexpr(self):
        return ("like", self.child.sexpr(), self.literal.decode("utf-8"), self.escape)


class In(_StringTest):
    """`child IN (values)` over string literals; a None among them makes a miss NULL instead of FALSE."""
    op, name = "STR_IN", "in"

    def __init__(self, child, values):
        super().__init__(child, b"")
        self.values = [None if v is None else _utf8(v) for v in values]

    def emit(self, schema, out):
        lits = [v for v in self.values if v is not None]
        blob = struct.pack("=I", len(lits)) + b"".join(struct.pack("=I", len(v)) + v for v in lits)
        out.append(_node(self.op, VT_BOOL, _string_col(self.child, schema), lit_i=_pool(out).slice(blob),
                         arg2=1 if None in self.values else 0))

    def sexpr(self):
        return ("in", self.child.sexpr(), list(self.values))


class OctetLength(_StringTest):
    op, name = "STR_OCTET_LENGTH", "octet_length"

    def __init__(self, child):
        super().__init__(child, b"")

    def vtype(self, schema):
        return VT_I32

    def emit(self, schema, out):
        out.append(_node(self.op, VT_I32, _string_col(self.child, schema)))

    def sexpr(self):
        return ("octet_length", self.child.sexpr())


class Length(OctetLength):
    """length(str): the code points, counted as UTF8String.numChars counts them (one per lead byte); over a binary column the bytes
    (stringExpressions.scala Length: `case BinaryType => value.length`)."""
    op, name = "STR_CHAR_LENGTH", "length"

    def emit(self, schema, out):
        i = _string_col(self.child, schema)
        out.append(_node("STR_OCTET_LENGTH" if self.child.name in schema.binary else self.op, VT_I32, i))

    def sexpr(self):
        return ("length", self.child.sexpr())


# ---- string-producing functions (stringExpressions.scala, collectionOperations.scala Concat) ----------------------------------
# Their value is a string, so they are programs of their own (SB_OP_SF_*, sb_string_project) rather than nodes of a numeric one.
# Positions, lengths and pad lengths are int literals; trim sets, pads and separators string literals; a None among them is a NULL
# literal and gives the function's NULL answer.  String operands are string columns, string literals or other string functions.
_INT_MAX = 2 ** 31 - 1
_ABSENT = object()


def _int_arg(v, what):
    if isinstance(v, Literal):
        v = v.value
    if v is None:
        return None
    if isinstance(v, bool) or not isinstance(v, int) or not -2 ** 31 <= v < 2 ** 31:
        raise capi.SparkB200Error(5, "%s must be an int literal (got %r)" % (what, v))
    return v


def _str_arg(v, what):
    if isinstance(v, Literal):
        v = v.value
    if v is None:
        return None
    if not isinstance(v, (str, bytes)):
        raise capi.SparkB200Error(5, "%s must be a string literal (got %r)" % (what, v))
    return _utf8(v)


def _string_operand(e):
    if isinstance(e, (str, bytes)) or e is None:
        return Literal(e, 0)
    if isinstance(e, Literal) and (e.value is None or isinstance(e.value, (str, bytes))):
        return Literal(e.value, 0)
    if isinstance(e, (AttributeReference, StringFunction)):
        return e
    raise capi.SparkB200Error(5, "string functions take string columns, string literals or string functions (got %r)" % (e,))


def _emit_sf_operand(e, schema, out):
    if isinstance(e, StringFunction):
        e.emit_sf(schema, out)
    elif isinstance(e, Literal):
        if e.value is None:
            out.append(_node("SF_LIT", 0, arg2=1))
        else:
            out.append(_node("SF_LIT", 0, lit_i=_pool(out).slice(_utf8(e.value))))
    else:
        out.append(_node("SF_COL", 0, _string_col(e, schema)))


def _sexpr_operand(e):
    return ("lit", e.value, bytes) if isinstance(e, Literal) else e.sexpr()


class StringFunction(Expression):
    name = None

    def vtype(self, schema):
        return 0

    def emit(self, schema, out):
        raise TypeError("%s yields a string: it is evaluated by sb_string_project, not inside a numeric program" % self.name)

    def emit_sf(self, schema, out):
        raise NotImplementedError


class Substring(StringFunction):
    """substring(str, pos[, len]) (UTF8String.substringSQL); len omitted = Integer.MAX_VALUE."""
    name = "substring"

    def __init__(self, child, pos, len=_INT_MAX):
        self.child = _string_operand(child)
        self.children = (self.child,)
        self.pos, self.len = _int_arg(pos, "substring position"), _int_arg(len, "substring length")

    def emit_sf(self, schema, out):
        if self.pos is None or self.len is None:
            out.append(_node("SF_LIT", 0, arg2=1))
            return
        _emit_sf_operand(self.child, schema, out)
        out.append(_node("SF_SUBSTRING", 0, self.pos, arg2=self.len))

    def sexpr(self):
        return ("substring", _sexpr_operand(self.child), self.pos, self.len)


class Concat(StringFunction):
    """concat(s1, s2, ...): NULL if any input is NULL."""
    name = "concat"

    def __init__(self, *children):
        self.children = tuple(_string_operand(c) for c in children)

    def emit_sf(self, schema, out):
        if not self.children:
            out.append(_node("SF_LIT", 0, lit_i=_pool(out).slice(b"")))
            return
        for c in self.children:
            _emit_sf_operand(c, schema, out)
        out.append(_node("SF_CONCAT", 0, len(self.children)))

    def sexpr(self):
        return ("concat",) + tuple(_sexpr_operand(c) for c in self.children)


class ConcatWs(StringFunction):
    """concat_ws(sep, s1, s2, ...): NULL inputs are skipped; a NULL separator gives NULL."""
    name = "concat_ws"

    def __init__(self, sep, *children):
        self.sep = _str_arg(sep, "concat_ws separator")
        self.children = tuple(_string_operand(c) for c in children)

    def emit_sf(self, schema, out):
        if self.sep is None:
            out.append(_node("SF_LIT", 0, arg2=1))
        elif not self.children:
            out.append(_node("SF_LIT", 0, lit_i=_pool(out).slice(b"")))
        else:
            for c in self.children:
                _emit_sf_operand(c, schema, out)
            out.append(_node("SF_CONCAT_WS", 0, len(self.children), lit_i=_pool(out).slice(self.sep)))

    def sexpr(self):
        return ("concat_ws", self.sep) + tuple(_sexpr_operand(c) for c in self.children)


class _Trim(StringFunction):
    op = None

    def __init__(self, srcStr, trimStr=_ABSENT):
        self.child = _string_operand(srcStr)
        self.children = (self.child,)
        self.given = trimStr is not _ABSENT
        self.trim = _str_arg(trimStr, "trim string") if self.given else None

    def emit_sf(self, schema, out):
        if self.given and self.trim is None:
            out.append(_node("SF_LIT", 0, arg2=1))
            return
        _emit_sf_operand(self.child, schema, out)
        if self.given:
            out.append(_node(self.op, 0, 1, lit_i=_pool(out).slice(self.trim)))
        else:
            out.append(_node(self.op, 0, 0))

    def sexpr(self):
        return (self.name, _sexpr_operand(self.child), self.trim if self.given else ())


class StringTrim(_Trim):
    """trim(str) removes ASCII spaces; trim(str, trimStr) every code point that occurs in trimStr, from both ends."""
    op, name = "SF_TRIM", "trim"


class StringTrimLeft(_Trim):
    op, name = "SF_LTRIM", "ltrim"


class StringTrimRight(_Trim):
    op, name = "SF_RTRIM", "rtrim"


class _Pad(StringFunction):
    op = None

    def __init__(self, str, len, pad=" "):
        self.child = _string_operand(str)
        self.children = (self.child,)
        self.len = _int_arg(len, "pad length")
        self.pad = _str_arg(pad, "pad")

    def emit_sf(self, schema, out):
        if self.len is None or self.pad is None:
            out.append(_node("SF_LIT", 0, arg2=1))
            return
        _emit_sf_operand(self.child, schema, out)
        out.append(_node(self.op, 0, self.len, lit_i=_pool(out).slice(self.pad)))

    def sexpr(self):
        return (self.name, _sexpr_operand(self.child), self.len, self.pad)


class StringLPad(_Pad):
    """lpad(str, len, pad): padding counted in code points."""
    op, name = "SF_LPAD", "lpad"


class StringRPad(_Pad):
    op, name = "SF_RPAD", "rpad"


class CompiledStringProgram:
    """Owns the ctypes arrays behind one string-producing sb_expr (SB_OP_SF_* nodes, out_type SB_STRING)."""

    def __init__(self, expr: Expression, schema: Schema):
        nodes = _Program()
        _emit_sf_operand(_string_operand(expr), schema, nodes)
        self.arr = (capi.sb_expr_node * len(nodes))(*nodes)
        self.c = capi.sb_expr()
        self.c.nodes = C.cast(self.arr, C.POINTER(capi.sb_expr_node))
        self.c.n = len(nodes)
        self.pool = (C.c_uint8 * max(1, len(nodes.pool))).from_buffer_copy(bytes(nodes.pool) or b"\0")
        self.c.bytes = C.cast(self.pool, C.c_void_p) if nodes.pool else None
        self.c.nbytes = len(nodes.pool)
        self.c.out_type = capi.SB_STRING


class CompiledExpr:
    """Owns the ctypes arrays behind one sb_expr: the nodes and the pool of string literals."""

    def __init__(self, expr: Expression, schema: Schema):
        nodes = _Program()
        expr.emit(schema, nodes)
        self.arr = (capi.sb_expr_node * len(nodes))(*nodes)
        self.c = capi.sb_expr()
        self.c.nodes = C.cast(self.arr, C.POINTER(capi.sb_expr_node))
        self.c.n = len(nodes)
        self.pool = (C.c_uint8 * max(1, len(nodes.pool))).from_buffer_copy(bytes(nodes.pool) or b"\0")
        self.c.bytes = C.cast(self.pool, C.c_void_p) if nodes.pool else None
        self.c.nbytes = len(nodes.pool)
        if isinstance(expr, AttributeReference):
            self.c.out_type = schema.types[schema.index(expr.name)]
        else:
            self.c.out_type = _OUT_OF_VT[expr.vtype(schema)]


# ---- aggregate functions (expressions/aggregate/{Sum,Average,Count,Min,Max}.scala) -----------------
class AggregateFunction:
    func = None

    def __init__(self, child=None):
        self.child = _wrap(child) if child is not None else None

    def sexpr_input(self):
        return None if self.child is None else self.child.sexpr()


class Sum(AggregateFunction):
    func = "sum"


class Average(AggregateFunction):
    func = "avg"


class Count(AggregateFunction):
    """Count(expr); Count() / Count(Literal(1)) is count(*)."""
    func = "count"

    def __init__(self, child=None):
        if child is None or (isinstance(child, Literal)) or isinstance(child, int):
            self.child = None
            self.func = "count_star"
        else:
            self.child = _wrap(child)


class Min(AggregateFunction):
    func = "min"


class Max(AggregateFunction):
    func = "max"


# ---- central moments (expressions/aggregate/CentralMomentAgg.scala:49-290) -------------------------------------------------
class _CentralMomentAgg(AggregateFunction):
    """Buffer (n, avg, m2), all doubles.  The input is cast to DOUBLE (ImplicitCastInputTypes); with
    null_on_divide_by_zero=False (spark.sql.legacy.statisticalAggregate) the _samp forms of one row give NaN, not NULL."""

    def __init__(self, child, null_on_divide_by_zero=True):
        super().__init__(Cast(_wrap(child), "double"))
        self.null_on_divide_by_zero = null_on_divide_by_zero


class StddevSamp(_CentralMomentAgg):
    """stddev_samp / stddev: sqrt(m2 / (n - 1))."""
    func = "stddev_samp"


class StddevPop(_CentralMomentAgg):
    func = "stddev_pop"


class VarianceSamp(_CentralMomentAgg):
    """var_samp / variance: m2 / (n - 1)."""
    func = "var_samp"


class VariancePop(_CentralMomentAgg):
    func = "var_pop"


Stddev, Variance = StddevSamp, VarianceSamp


class SortOrder:
    """SortOrder(child, direction, nullOrdering) (SortOrder.scala:63); default null ordering: ASC -> NULLS
    FIRST, DESC -> NULLS LAST."""

    def __init__(self, child, ascending=True, nulls_first=None):
        self.child = child if isinstance(child, str) else child.name
        self.ascending = ascending
        self.nulls_first = ascending if nulls_first is None else nulls_first

    def as_tuple(self):
        return (self.child, self.ascending, self.nulls_first)
