"""UDF front end: Python lambdas/defs -> tplx op program (include/tplx_ir.h).

Stands where the reference's codegen stands (tuplex/codegen: ASTBuilderVisitor, TypeAnnotatorVisitor,
BlockGeneratorVisitor, FunctionRegistry; driven by StageBuilder::generateFastCodePath,
tuplex/core/src/physical/StageBuilder.cc:602-1143) but emits a flat predicated register program
instead of LLVM IR. Typing is static from the normal-case input schema, like the reference's
TypeAnnotatorVisitor. Anything outside the supported op set raises UnsupportedUDF; the caller then
routes the operator's rows to the CPython path (the reference does the same when a UDF cannot be
compiled: it falls back to the interpreter, tuplex/python/tuplex/dataset.py:49-80).

Python control flow is if-converted: every instruction carries a guard, `if/elif/else` and early
`return` become guards + SEL, so instructions of untaken branches can never raise
(reference semantics: an exception is only raised on the executed path, PipelineBuilder.cc:949).
"""
from __future__ import annotations

import ast
import inspect
import linecache
import re
import types
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Sequence, Tuple, Union

from . import ir
from .ir import C, Instr, NOSLOT, Program, T_BOOL, T_F64, T_I64, T_STR


class UnsupportedUDF(Exception):
    """The UDF uses something outside the GPU op set -> CPython path."""


# ------------------------------------------------------------------------------------------------
# locating the AST of a function object
# ------------------------------------------------------------------------------------------------
_file_ast_cache: Dict[str, Tuple[int, ast.AST]] = {}


def _file_ast(filename: str) -> Optional[ast.AST]:
    lines = linecache.getlines(filename)
    if not lines:
        return None
    key = hash(tuple(lines))
    hit = _file_ast_cache.get(filename)
    if hit and hit[0] == key:
        return hit[1]
    try:
        tree = ast.parse("".join(lines), filename)
    except SyntaxError:
        return None
    _file_ast_cache[filename] = (key, tree)
    return tree


def _code_signature(code: types.CodeType):
    consts = tuple(c for c in code.co_consts if not isinstance(c, types.CodeType))
    return (code.co_code, consts, code.co_names, code.co_varnames[: code.co_argcount])


def get_udf_ast(func) -> Tuple[List[str], Union[ast.expr, List[ast.stmt]], Dict[str, Any]]:
    """Return (argument names, body, resolvable globals/closure) for a lambda or def."""
    if isinstance(func, str):  # source string, like the reference's UDF("lambda x: ...") / UDF("def f(x):\n ...") in C++ tests
        src = func.strip()
        if src.startswith("def "):
            import textwrap
            mod = ast.parse(textwrap.dedent(func).strip().expandtabs(4))
            fns = [n for n in mod.body if isinstance(n, ast.FunctionDef)]
            if len(fns) != 1:
                raise UnsupportedUDF("UDF string must hold one function")
            _check_args(fns[0].args)
            return [a.arg for a in fns[0].args.args], fns[0].body, {}
        node = ast.parse(src, mode="eval").body
        if not isinstance(node, ast.Lambda):
            raise UnsupportedUDF("UDF string must be a lambda or a def")
        return [a.arg for a in node.args.args], node.body, {}
    if not isinstance(func, types.FunctionType):
        raise UnsupportedUDF(f"not a plain Python function: {func!r}")
    code = func.__code__
    env: Dict[str, Any] = dict(func.__globals__)
    if func.__closure__:
        for name, cell in zip(code.co_freevars, func.__closure__):
            try:
                env[name] = cell.cell_contents
            except ValueError:
                pass
    tree = _file_ast(code.co_filename)
    if tree is None:
        raise UnsupportedUDF("source of UDF not available")
    if code.co_name == "<lambda>":
        cands = [n for n in ast.walk(tree) if isinstance(n, ast.Lambda) and n.lineno <= code.co_firstlineno <= (n.end_lineno or n.lineno)]
        cands = [n for n in cands if n.lineno == code.co_firstlineno] or cands
        if len(cands) > 1:
            sig = _code_signature(code)
            matched = []
            for n in cands:
                try:
                    mod = compile(ast.Expression(body=n), code.co_filename, "eval")
                    inner = [c for c in mod.co_consts if isinstance(c, types.CodeType)]
                    if inner and _code_signature(inner[0]) == sig:
                        matched.append(n)
                except Exception:
                    continue
            if matched:
                cands = matched[:1]
        if len(cands) != 1:
            raise UnsupportedUDF("cannot locate lambda source unambiguously")
        node = cands[0]
        _check_args(node.args)
        return [a.arg for a in node.args.args], node.body, env
    for n in ast.walk(tree):
        if isinstance(n, ast.FunctionDef) and n.name == code.co_name and n.lineno <= code.co_firstlineno + len(n.decorator_list) + 1 \
                and (n.end_lineno or n.lineno) >= code.co_firstlineno:
            _check_args(n.args)
            return [a.arg for a in n.args.args], n.body, env
    raise UnsupportedUDF("cannot locate function source")


def _check_args(a: ast.arguments):
    if a.vararg or a.kwarg or a.kwonlyargs or a.defaults or a.posonlyargs:
        raise UnsupportedUDF("only plain positional parameters are supported")


# ------------------------------------------------------------------------------------------------
# compile-time values
# ------------------------------------------------------------------------------------------------
@dataclass
class Val:
    """A typed scalar/string value: either a compile-time constant or a virtual register."""
    type: int
    vreg: Optional[int] = None
    const: Any = None
    sel: Any = None  # (cond, a, b) when this value is cond ? a : b
    null: Any = None  # Option[T] value: bool Val "this row's value is None" (None = the value can never be None)

    @property
    def is_const(self):
        return self.vreg is None


@dataclass
class TupleVal:
    elems: List[Any]  # Val | TupleVal
    names: Optional[List[Optional[str]]] = None
    is_list: bool = False


def _py_type_of(v) -> int:
    if isinstance(v, bool):
        return T_BOOL
    if isinstance(v, int):
        return T_I64
    if isinstance(v, float):
        return T_F64
    if isinstance(v, str):
        return T_STR
    raise UnsupportedUDF(f"unsupported constant {v!r}")


def const_val(v) -> Val:
    return Val(_py_type_of(v), None, v)


T_NONE = -1  # static type of the literal None (python::Type::NULLVALUE): a value that is None for every row


def none_val() -> Val:
    return Val(T_NONE, None, None, None, const_val(True))


def is_none_literal(v) -> bool:
    return isinstance(v, Val) and v.type == T_NONE


def plain(v: Val) -> Val:
    """The same value without its None flag (callers have dealt with the None rows)."""
    if v.null is None:
        return v
    return Val(v.type, v.vreg, v.const, v.sel)


# ------------------------------------------------------------------------------------------------
# the stage compiler
# ------------------------------------------------------------------------------------------------
class StageCompiler:
    """Accumulates the operators of one stage and emits a Program.

    Mirrors PipelineBuilder's per-operator API (tuplex/core/src/physical/PipelineBuilder.cc:
    mapOperation :565, filterOperation :615, mapColumnOperation :706, withColumnOperation :808,
    addAggregate :2525, buildWithHashmapWriter :1108).
    """

    def __init__(self, in_types: Sequence[int], in_names: Sequence[Optional[str]], option_cols: Sequence[int] = ()):
        """option_cols: input columns of type Option[T] (normal case with None values, utils/include/TypeSystem.h; the reference keeps
        a per-row bitmap for them, Serializer.cc:1041-1059). Each gets an "is None" companion input column of type bool behind the
        physical columns (descriptor: in_types entry TPLX_T_NULLOF | column); the executor expands the column's validity bitmap into
        it. UDF code sees a value with a None flag: `is None` / `== None` tests read the flag, any other use of a None value raises
        TypeError for that row (it is resolved on the interpreter path), values flow to the output with their flag."""
        in_types, in_names = list(in_types), list(in_names)
        self.phys_types, self.phys_names = list(in_types), list(in_names)
        self.option_cols = sorted(set(int(c) for c in option_cols))
        null_of = {len(in_types) + k: c for k, c in enumerate(self.option_cols)}
        self.prog = Program(in_types + [T_BOOL] * len(null_of), in_names + [None] * len(null_of))
        self.prog.null_of = dict(null_of)
        self.vreg_width: List[int] = []
        self.row: List[Val] = []
        self.names: List[Optional[str]] = list(in_names)
        self._col_cache: Dict[int, Val] = {}
        self.cur_op = 0
        self.guard: Optional[int] = None  # vreg of current guard
        self.filters: List[Tuple[int, int]] = []  # (pc after the FILTER instruction, number of logged operators incl. it)
        self.oplog: List[Tuple[str, tuple]] = []  # operators in order, so that a prefix can be replayed (prefilter stage)
        comp = {c: j for j, c in null_of.items()}
        for c, t in enumerate(in_types):
            v = Val(t, None, ("col", c))  # lazily loaded column reference
            if c in comp:
                v.null = Val(T_BOOL, None, ("col", comp[c]))
            self.row.append(v)

    # ---- emission helpers ----------------------------------------------------------------------
    def new_vreg(self, t: int) -> int:
        self.vreg_width.append(2 if t == T_STR else 1)
        return len(self.vreg_width) - 1

    def emit(self, op, dst=None, a=None, b=None, c=None, flags=0, imm=0, imm2=0) -> None:
        def r(x):
            return NOSLOT if x is None else x
        self.prog.instrs.append(Instr(op, r(dst), r(a), r(b), r(c), r(self.guard), self.cur_op, flags, imm, imm2))

    def reg(self, v: Val) -> int:
        """Materialise a value into a vreg (loads constants / columns on demand)."""
        if v.vreg is not None:
            return v.vreg
        if isinstance(v.const, tuple) and v.const and v.const[0] == "col":
            col = v.const[1]
            hit = self._col_cache.get(col)
            if hit is not None:
                v.vreg = hit.vreg
                return v.vreg
            # column loads are hoisted out of any guard: they cannot raise and must dominate all uses
            g, self.guard = self.guard, None
            d = self.new_vreg(v.type)
            self.emit(C["TPLX_OP_LDCOL"], d, flags=v.type, imm=col)
            self.guard = g
            v.vreg = d
            self._col_cache[col] = v
            return d
        d = self.new_vreg(v.type)
        g, self.guard = self.guard, None  # constants are unconditional
        if v.type == T_STR:
            self.emit(C["TPLX_OP_LDS"], d, imm=self._enc_const(v))
        elif v.type == T_F64:
            self.emit(C["TPLX_OP_LDI"], d, imm=ir.f64_bits(float(v.const)))
        else:
            self.emit(C["TPLX_OP_LDI"], d, imm=int(v.const) & ((1 << 64) - 1))
        self.guard = g
        return d

    def _is_colref(self, v: Val) -> bool:
        return v.vreg is None and isinstance(v.const, tuple) and bool(v.const) and v.const[0] == "col"

    def is_const(self, v) -> bool:
        return isinstance(v, Val) and v.vreg is None and not self._is_colref(v)

    def _enc_const(self, v: Val) -> int:
        """Immediate encoding of a compile-time constant operand (include/tplx_ir.h tplx_constflag)."""
        if v.type == T_STR:
            off, ln = self.prog.const_bytes(v.const.encode("utf-8"))
            return off | (ln << 32)
        if v.type == T_F64:
            return ir.f64_bits(float(v.const))
        return int(v.const) & ((1 << 64) - 1)

    _NO_CONST_OPS = None

    def emit_vals(self, op, dst, a: Optional[Val] = None, b: Optional[Val] = None, c: Optional[Val] = None, flags=0, imm=0):
        """Emit an instruction whose operands are Vals; compile-time constants ride in the immediates
        (a <- imm2, b <- imm, c <- imm2) instead of being loaded into slots for every row."""
        if StageCompiler._NO_CONST_OPS is None:
            StageCompiler._NO_CONST_OPS = {C[k] for k in ("TPLX_OP_FILTER", "TPLX_OP_SFMTD", "TPLX_OP_I2S", "TPLX_OP_LDCOL", "TPLX_OP_LDI",
                                                             "TPLX_OP_LDS", "TPLX_OP_LDROW", "TPLX_OP_RAISE")}
        imm2 = 0
        ra = rb_ = rc = None
        ok = op not in StageCompiler._NO_CONST_OPS
        if b is not None:
            if ok and self.is_const(b):
                flags |= C["TPLX_F_B_CONST"]
                imm = self._enc_const(b)
            else:
                rb_ = self.reg(b)
        c_const = c is not None and ok and self.is_const(c) and op != C["TPLX_OP_SEL"]
        if c is not None:
            if c_const:
                flags |= C["TPLX_F_C_CONST"]
                imm2 = self._enc_const(c)
            else:
                rc = self.reg(c)
        if a is not None:
            if ok and self.is_const(a) and not c_const:
                flags |= C["TPLX_F_A_CONST"]
                imm2 = self._enc_const(a)
            else:
                ra = self.reg(a)
        self.emit(op, dst, ra, rb_, rc, flags=flags, imm=imm, imm2=imm2)

    def op2(self, op, t, a: Val, b: Val, flags=0) -> Val:
        d = self.new_vreg(t)
        self.emit_vals(op, d, a, b, flags=flags)
        return Val(t, d)

    def op1(self, op, t, a: Val, flags=0, imm=0) -> Val:
        d = self.new_vreg(t)
        self.emit_vals(op, d, a, flags=flags, imm=imm)
        return Val(t, d)

    # ---- type coercions (BlockGeneratorVisitor upCast) -----------------------------------------
    def to_f64(self, v: Val) -> Val:
        if v.type == T_F64:
            return v
        if v.type in (T_I64, T_BOOL):
            if self.is_const(v):
                return const_val(float(int(v.const)))
            return self.op1(C["TPLX_OP_I2F"], T_F64, v)
        raise UnsupportedUDF("cannot convert str to float implicitly")

    def to_i64(self, v: Val) -> Val:
        if v.type == T_I64:
            return v
        if v.type == T_BOOL:
            if self.is_const(v):
                return const_val(int(v.const))
            return Val(T_I64, self.reg(v))  # bool is stored as 0/1
        raise UnsupportedUDF("expected integer")

    def truth(self, v) -> Val:
        """Python truth value test (LLVMEnvironment::truthValueTest; filter: PipelineBuilder.cc:671-686)."""
        if isinstance(v, TupleVal):
            return const_val(len(v.elems) > 0)
        if v.null is not None:  # None is false; a value is tested as usual
            if v.type == T_NONE:
                return const_val(False)
            return self.b_and(self.b_not(v.null), self.truth(plain(v)))
        if self.is_const(v):
            return const_val(bool(v.const))
        if v.type == T_BOOL:
            return v
        if v.type == T_I64:
            return self.op2(C["TPLX_OP_ICMP"], T_BOOL, v, const_val(0), flags=C["TPLX_CMP_NE"])
        if v.type == T_F64:
            return self.op2(C["TPLX_OP_FCMP"], T_BOOL, v, const_val(0.0), flags=C["TPLX_CMP_NE"])
        return self.op1(C["TPLX_OP_STRUTH"], T_BOOL, v)

    def b_and(self, a: Optional[Val], b: Val) -> Val:
        if a is None:
            return b
        if self.is_const(a):
            return b if a.const else const_val(False)
        if self.is_const(b):
            return a if b.const else const_val(False)
        return self.op2(C["TPLX_OP_BAND"], T_BOOL, a, b)

    def b_or(self, a: Val, b: Val) -> Val:
        if self.is_const(a):
            return const_val(True) if a.const else b
        if self.is_const(b):
            return const_val(True) if b.const else a
        return self.op2(C["TPLX_OP_BOR"], T_BOOL, a, b)

    def b_not(self, a: Val) -> Val:
        if self.is_const(a):
            return const_val(not a.const)
        return self.op1(C["TPLX_OP_BNOT"], T_BOOL, a)

    def select(self, cond: Val, a, b):
        """cond ? a : b over scalars and tuples."""
        if isinstance(a, TupleVal) or isinstance(b, TupleVal):
            if not (isinstance(a, TupleVal) and isinstance(b, TupleVal) and len(a.elems) == len(b.elems)):
                raise UnsupportedUDF("branches return different shapes")
            return TupleVal([self.select(cond, x, y) for x, y in zip(a.elems, b.elems)], a.names or b.names)
        if self.is_const(cond):
            return a if cond.const else b
        if a.null is not None or b.null is not None:
            # Option[T]: select the values and the None flags separately (upCastReturnType, BlockGeneratorVisitor.cc:4055-4075)
            if a.type == T_NONE and b.type == T_NONE:
                return a
            zero = {T_STR: "", T_F64: 0.0, T_BOOL: False}
            na = a.null if a.null is not None else const_val(False)
            nb = b.null if b.null is not None else const_val(False)
            va = plain(a) if a.type != T_NONE else const_val(zero.get(b.type, 0))
            vb = plain(b) if b.type != T_NONE else const_val(zero.get(a.type, 0))
            out = self.select(cond, va, vb)
            null = self.select(cond, na, nb)
            if self.is_const(null) and not null.const:
                return out
            return Val(out.type, out.vreg, out.const, out.sel, null)
        a, b = self.unify(a, b)
        if a.type == T_BOOL:
            # boolean selects with constant arms are plain logic
            if self.is_const(a) and self.is_const(b):
                return a if bool(a.const) == bool(b.const) else (cond if a.const else self.b_not(cond))
            if self.is_const(a):
                return self.b_or(cond, b) if a.const else self.b_and(self.b_not(cond), b)
            if self.is_const(b):
                return self.b_or(self.b_not(cond), a) if b.const else self.b_and(cond, a)
        d = self.new_vreg(a.type)
        # SEL itself must run wherever either side may be needed later: emit under the current guard
        self.emit_vals(C["TPLX_OP_SEL"], d, a, b, cond, flags=2 if a.type == T_STR else 1)
        out = Val(a.type, d)
        out.sel = (cond, a, b)  # provenance: lets comparisons against constants fold through the select
        return out

    def unify(self, a: Val, b: Val) -> Tuple[Val, Val]:
        if a.type == b.type:
            return a, b
        nums = (T_I64, T_BOOL)
        if a.type in nums and b.type in nums:
            return self.to_i64(a), self.to_i64(b)
        raise UnsupportedUDF("branches produce different types (normal case must be uniformly typed)")

    # ---- pipeline operators ----------------------------------------------------------------------
    def begin_op(self, op_id: int):
        self.prog.opids.append(int(op_id))
        self.cur_op = len(self.prog.opids) - 1
        self.guard = None

    def row_value(self):
        if len(self.row) == 1:
            return self.row[0]
        return TupleVal(list(self.row), list(self.names))

    def _call_udf(self, func, args_vals: List[Any]):
        argnames, body, env = get_udf_ast(func)
        if len(argnames) != len(args_vals):
            # Tuplex unpacks a tuple row over multiple lambda parameters
            if len(args_vals) == 1 and isinstance(args_vals[0], TupleVal) and len(args_vals[0].elems) == len(argnames):
                args_vals = list(args_vals[0].elems)
            else:
                raise UnsupportedUDF("UDF arity does not match row")
        fc = _FuncCompiler(self, env)
        return fc.run(argnames, args_vals, body)

    def add_map(self, func, op_id: int):
        self.oplog.append(("add_map", (func, op_id)))
        self.begin_op(op_id)
        res = self._call_udf(func, [self.row_value()])
        if isinstance(res, TupleVal) and res.is_list:
            raise UnsupportedUDF("list-valued map output")
        if isinstance(res, TupleVal):
            flat, names = [], []
            for i, e in enumerate(res.elems):
                if isinstance(e, TupleVal):
                    raise UnsupportedUDF("nested tuples in map output")
                flat.append(e)
                names.append(res.names[i] if res.names else None)
            self.row, self.names = flat, names
        else:
            self.row, self.names = [res], [None]

    def add_filter(self, func, op_id: int):
        self.oplog.append(("add_filter", (func, op_id)))
        self.begin_op(op_id)
        res = self.truth(self._call_udf(func, [self.row_value()]))
        self.guard = None
        self.emit(C["TPLX_OP_FILTER"], a=self.reg(res))
        self.filters.append((len(self.prog.instrs), len(self.oplog)))

    def col_index(self, key) -> int:
        if isinstance(key, int):
            if not -len(self.row) <= key < len(self.row):
                raise UnsupportedUDF("column index out of range")
            return key % len(self.row)
        if key not in self.names:
            raise UnsupportedUDF(f"unknown column {key!r}")
        return self.names.index(key)

    def add_with_column(self, name: str, func, op_id: int):
        self.oplog.append(("add_with_column", (name, func, op_id)))
        self.begin_op(op_id)
        res = self._call_udf(func, [self.row_value()])
        if isinstance(res, TupleVal):
            raise UnsupportedUDF("withColumn UDF must return a scalar")
        if name in self.names:
            self.row[self.names.index(name)] = res
        else:
            self.row.append(res)
            self.names.append(name)

    def add_map_column(self, name, func, op_id: int):
        self.oplog.append(("add_map_column", (name, func, op_id)))
        self.begin_op(op_id)
        i = self.col_index(name)
        res = self._call_udf(func, [self.row[i]])
        if isinstance(res, TupleVal):
            raise UnsupportedUDF("mapColumn UDF must return a scalar")
        self.row[i] = res

    def add_select(self, cols: Sequence[Union[int, str]], op_id: int):
        self.oplog.append(("add_select", (cols, op_id)))
        self.begin_op(op_id)
        idx = [self.col_index(c) for c in cols]
        self.row = [self.row[i] for i in idx]
        self.names = [self.names[i] for i in idx]

    def add_rename(self, old, new: str, op_id: int):
        self.oplog.append(("add_rename", (old, new, op_id)))
        self.begin_op(op_id)
        self.names[self.col_index(old)] = new

    # ---- endpoints ---------------------------------------------------------------------------------
    def _finish(self, used_vals: List[Val]) -> List[int]:
        self.guard = None
        regs = [self.reg(v) for v in used_vals]
        self._dce(regs)
        self._fuse(regs)   # idioms first: they are recognised in the guarded form the if-conversion emits
        self._cse(regs)
        self._dce(regs)
        if getattr(self, "_want_scan_hint", False):
            self.prog.fused = _match_string_scan(self)  # closed form of a pure filter chain (None when it is not one)
        slots = self._regalloc(regs)
        return slots

    def _cse(self, live_out: List[int]):
        """Common-subexpression elimination on the single-assignment vreg program (what LLVM's GVN does for the reference,
        LLVMOptimizer.cc:119-191). If-conversion of early returns recomputes the same path conditions (`not done`, `a and not done`)
        for every statement; two passes:
          1. a cheap, non-raising instruction whose operands are defined for every row loses its guard (its result is then defined
             for every row too; rows outside the guard never look at it);
          2. identical unguarded pure instructions share one result."""
        ins = self.prog.instrs
        OP = lambda k: C["TPLX_OP_" + k]
        ndef: Dict[int, int] = {}
        for i in ins:
            if i.dst != NOSLOT:
                ndef[i.dst] = ndef.get(i.dst, 0) + 1
        cheap = {OP(k) for k in ("BNOT", "BAND", "BOR", "ICMP", "FCMP", "IADD", "ISUB", "IMUL", "INEG", "IAND", "IOR", "IXOR", "IABS", "FADD", "FSUB",
                                 "FMUL", "FNEG", "FABS", "I2F", "SEL", "SLEN", "SLOWER", "SUPPER", "STRUTH", "SSLICE", "SEQ", "LDI", "LDS")}
        pure = cheap | {OP(k) for k in ("SFIND", "SRFIND", "SIN", "SSTARTS", "SENDS", "SSTRIP", "ISHL", "ISHR", "F2I", "SFINDE", "SRFINDK", "LDROW")}
        everywhere = set()  # vregs that hold a defined value for every row
        for i in ins:
            ops = [r for r in (i.a, i.b, i.c) if r != NOSLOT]
            single = i.dst != NOSLOT and ndef.get(i.dst, 0) == 1
            if i.guard != NOSLOT and single and i.op in cheap and i.guard in everywhere and all(r in everywhere for r in ops):
                i.guard = NOSLOT
            if i.guard == NOSLOT and single and all(r in everywhere for r in ops):
                everywhere.add(i.dst)
        seen: Dict[tuple, int] = {}
        repl: Dict[int, int] = {}
        out = []
        keep = set(live_out)
        for i in ins:
            for f in ("a", "b", "c", "guard"):
                v = getattr(i, f)
                if v in repl:
                    setattr(i, f, repl[v])
            if (i.guard == NOSLOT and i.dst != NOSLOT and ndef.get(i.dst, 0) == 1 and i.op in pure and i.dst not in keep
                    and all(r == NOSLOT or ndef.get(r, 0) == 1 for r in (i.a, i.b, i.c))):
                key = (i.op, i.flags, i.a, i.b, i.c, i.imm, i.imm2, self.vreg_width[i.dst])
                if key in seen:
                    repl[i.dst] = seen[key]
                    continue
                seen[key] = i.dst
            out.append(i)
        self.prog.instrs[:] = out

    def _fuse(self, live_out: List[int]):
        """Peephole fusion on the (single-assignment) vreg program: two idioms that every 'split at a marker' UDF
        produces become one instruction each (include/tplx_ir.h TPLX_OP_SFINDE / TPLX_OP_SRFINDK). Each fused op is
        defined as the primitive sequence it replaces, which is what the oracle evaluates; the reference gets the same
        effect from LLVM's inlining + select folding (tuplex/core/src/physical/LLVMOptimizer.cc:119-191).
          i = s.find(m);  stop = len(s) if i < 0 else i          -> SFINDE
          i = s.rfind(m); start = 0 if i < 0 else i + K          -> SRFINDK"""
        ins = self.prog.instrs
        ndef: Dict[int, int] = {}
        nuse: Dict[int, int] = {}
        where: Dict[int, int] = {}
        for pc, i in enumerate(ins):
            if i.dst != NOSLOT:
                ndef[i.dst] = ndef.get(i.dst, 0) + 1
                where[i.dst] = pc
            for r in (i.a, i.b, i.c, i.guard):
                if r != NOSLOT:
                    nuse[r] = nuse.get(r, 0) + 1
        for r in live_out:
            nuse[r] = nuse.get(r, 0) + 1
        OP = lambda k: C["TPLX_OP_" + k]
        AC, BC = C["TPLX_F_A_CONST"], C["TPLX_F_B_CONST"]

        def single(v):
            return v != NOSLOT and ndef.get(v, 0) == 1

        def d(v):
            return ins[where[v]] if single(v) else None

        def stable(v):  # operand may be read later than where it was read originally
            return v == NOSLOT or ndef.get(v, 0) == 1

        def is_lt0(ci, xv):
            return (ci is not None and ci.op == OP("ICMP") and ci.a == xv and (ci.flags & BC) and not (ci.flags & AC)
                    and (ci.flags & 7) == C["TPLX_CMP_LT"] and ci.imm == 0 and ci.guard == NOSLOT)

        dead = set()
        for y in ins:
            if y.op != OP("SEL") or (y.flags & 3) != 1 or y.guard != NOSLOT or not single(y.dst) or y.c == NOSLOT:
                continue
            cv = y.c
            ci = d(cv)
            if ci is None:
                continue
            if not (y.flags & (AC | BC)) and y.a != NOSLOT and y.b != NOSLOT:
                # SEL(c ? len(s) : x),  x = find(s, m), c = x < 0, len(s) guarded by c
                xi, li = d(y.b), d(y.a)
                if (xi is not None and li is not None and xi.op == OP("SFIND") and li.op == OP("SLEN") and is_lt0(ci, y.b)
                        and xi.guard == NOSLOT and li.guard == cv and li.a == xi.a and xi.a != NOSLOT and not (xi.flags & AC)
                        and stable(xi.a) and stable(xi.b) and nuse.get(y.b, 0) == 2 and nuse.get(cv, 0) == 2 and nuse.get(y.a, 0) == 1):
                    y.op, y.a, y.b, y.c = OP("SFINDE"), xi.a, xi.b, NOSLOT
                    y.flags, y.imm, y.imm2 = xi.flags & BC, xi.imm, 0
                    dead.update(id(k) for k in (xi, ci, li))
            elif (y.flags & AC) and not (y.flags & BC) and y.imm2 == 0 and y.b != NOSLOT:
                # SEL(c ? 0 : z),  z = x + K under !c,  x = rfind(s, m), c = x < 0
                zi = d(y.b)
                if zi is None or zi.op != OP("IADD") or not (zi.flags & BC) or (zi.flags & AC) or zi.guard == NOSLOT:
                    continue
                nci, xi = d(zi.guard), d(zi.a)
                if (nci is not None and xi is not None and nci.op == OP("BNOT") and nci.a == cv and nci.guard == NOSLOT
                        and xi.op == OP("SRFIND") and xi.guard == NOSLOT and xi.a != NOSLOT and not (xi.flags & AC) and is_lt0(ci, zi.a)
                        and stable(xi.a) and stable(xi.b) and nuse.get(zi.a, 0) == 2 and nuse.get(cv, 0) == 2
                        and nuse.get(zi.guard, 0) == 1 and nuse.get(y.b, 0) == 1):
                    y.op, y.a, y.b, y.c = OP("SRFINDK"), xi.a, xi.b, NOSLOT
                    y.flags, y.imm, y.imm2 = xi.flags & BC, xi.imm, zi.imm
                    dead.update(id(k) for k in (xi, ci, nci, zi))
        if dead:
            self.prog.instrs[:] = [i for i in ins if id(i) not in dead]

    def _dce(self, live_out: List[int]):
        """Drop pure instructions whose result is never used. Instructions that can raise or that steer rows
        (FILTER) always stay, so exception behaviour is unchanged (the reference's LLVM -O2 removes the same dead
        code, tuplex/core/src/physical/LLVMOptimizer.cc:119-191)."""
        side = {C[k] for k in ("TPLX_OP_FILTER", "TPLX_OP_RAISE", "TPLX_OP_IFLOORDIV", "TPLX_OP_IMOD", "TPLX_OP_FDIV", "TPLX_OP_FMOD",
                               "TPLX_OP_FFLOORDIV", "TPLX_OP_SINDEX", "TPLX_OP_S2I", "TPLX_OP_S2F")}
        live = set(live_out)
        keep = []
        for ins in reversed(self.prog.instrs):
            if ins.op in side or (ins.dst != NOSLOT and ins.dst in live):
                keep.append(ins)
                for r in (ins.a, ins.b, ins.c, ins.guard):
                    if r != NOSLOT:
                        live.add(r)
        keep.reverse()
        self.prog.instrs[:] = keep

    def finish_memory(self, prefilter: bool = True, scan_hint: bool = False) -> Program:
        self.prog.endpoint = C["TPLX_EP_MEMORY"]
        self._want_scan_hint = scan_hint
        n_user = len(self.row)
        k = self._choose_split() if prefilter else 0
        if k:
            # selective pipeline: a prefilter stage finds the surviving rows, this stage then runs densely over
            # them. The hidden trailing column (input row index of each output row) lets the executor number
            # exception rows across the two launches.
            pre = StageCompiler(self.phys_types, self.phys_names, self.option_cols)
            for name, a in self.oplog[:k]:
                getattr(pre, name)(*a)
            pre.begin_op(self.oplog[k - 1][1][-1])
            d = pre.new_vreg(T_I64)
            pre.emit(C["TPLX_OP_LDROW"], d)
            pre.row, pre.names = [Val(T_I64, d)], ["__row"]
            self.prog.prefilter = pre.finish_memory(prefilter=False, scan_hint=True)
            self.begin_op(self.oplog[-1][1][-1] if self.oplog else 0)
            d = self.new_vreg(T_I64)
            self.emit(C["TPLX_OP_LDROW"], d)
            self.row.append(Val(T_I64, d))
            self.names.append("__row")
            self.prog.hidden_out_cols = 1
        # Option[T] outputs: the value column plus a hidden bool "is None" companion (descriptor: tplx_outcol.null_of); the executor
        # packs the companion into the result's validity bitmap. Companions sit behind the visible columns, before "__row".
        outs, null_of = [], []
        for i, v in enumerate(self.row[:n_user]):
            if v.type == T_NONE:
                raise UnsupportedUDF("a column that is None for every row is not a normal-case column")
            outs.append(plain(v))
            null_of.append(0)
        comps = [(i, v.null) for i, v in enumerate(self.row[:n_user]) if v.null is not None and not (self.is_const(v.null) and not v.null.const)]
        for i, nv in comps:
            outs.append(nv)
            null_of.append(i + 1)
        outs += self.row[n_user:]
        null_of += [0] * (len(self.row) - n_user)
        self.prog.hidden_out_cols += len(comps)
        slots = self._finish(outs)
        self.prog.out_cols = [(s, v.type) for s, v in zip(slots, outs)]
        self.prog.out_null_of = null_of
        self.prog.out_names = list(self.names[:n_user])
        if k:
            self.row.pop()
            self.names.pop()
        return self.prog

    def _choose_split(self) -> int:
        """Number of leading operators to put into a prefilter stage (0 = none): the last filter that still has
        heavy work behind it. Late materialisation: everything behind it only touches surviving rows."""
        heavy = {C[k] for k in ("TPLX_OP_SREPLACE", "TPLX_OP_SCONCAT", "TPLX_OP_SFMTD", "TPLX_OP_SFIND", "TPLX_OP_SRFIND",
                                "TPLX_OP_S2I", "TPLX_OP_SIN", "TPLX_OP_I2S")}
        best = 0
        for pc, nops in self.filters:
            rest = self.prog.instrs[pc:]
            if rest and (sum(1 for i in rest if i.op in heavy) >= 2 or len(rest) >= 24):
                best = nops
        return best

    def finish_aggregate(self, agg_func, combine_func, init, op_id: int) -> Program:
        """aggregate(combine, agg, init) -> AGG_GENERAL endpoint (AggregateFunctions.cc:16-243)."""
        try:
            self.prog.fused = _match_fused_scan_aggregate(self, agg_func, combine_func, init)
        except UnsupportedUDF:
            self.prog.fused = None
        self.begin_op(op_id)
        accs = self._lower_aggregate(agg_func, combine_func, init)
        self.prog.endpoint = C["TPLX_EP_AGGREGATE"]
        slots = self._finish([v for _, v, _ in accs])
        self.prog.accs = [ir.Acc(kind, s, bits) for (kind, _, bits), s in zip(accs, slots)]
        self.prog.out_cols = []
        return self.prog

    def finish_hash(self, key_cols: Sequence[Union[int, str]], agg_func, combine_func, init, op_id: int) -> Program:
        """aggregateByKey / unique (PipelineBuilder.cc:1108-1400). An Option[T] key keeps None as a group of its own (the reference's
        null bucket, PipelineBuilder.cc:1148-1170,1263-1310): its "is None" flag goes out as a hidden bool column behind the keys
        (descriptor: tplx_outcol.null_of), and the device result carries the key column with a validity bitmap."""
        self.begin_op(op_id)
        kidx = [self.col_index(k) for k in key_cols]
        for i in kidx:
            if self.row[i].type == T_NONE:
                raise UnsupportedUDF("a key column that is None for every row is not a normal-case column")
            if self.row[i].type not in (T_I64, T_STR, T_BOOL):
                raise UnsupportedUDF("f64 keys are not supported (reference: PipelineBuilder.cc:1175-1177)")
        accs = self._lower_aggregate(agg_func, combine_func, init) if agg_func is not None else []
        self.prog.endpoint = C["TPLX_EP_HASH"]
        keys = [plain(self.row[i]) for i in kidx]
        comps = [(k, self.row[i].null) for k, i in enumerate(kidx)
                 if self.row[i].null is not None and not (self.is_const(self.row[i].null) and not self.row[i].null.const)]
        slots = self._finish(keys + [nv for _, nv in comps] + [v for _, v, _ in accs])
        self.prog.n_keys = len(keys)
        self.prog.out_cols = [(s, v.type) for s, v in zip(slots[: len(keys)], keys)]
        if comps:
            self.prog.out_cols += [(s, T_BOOL) for s in slots[len(keys): len(keys) + len(comps)]]
            self.prog.out_null_of = [0] * len(keys) + [k + 1 for k, _ in comps]
            self.prog.hidden_out_cols = len(comps)
            slots = slots[: len(keys)] + slots[len(keys) + len(comps):]
        self.prog.out_names = [self.names[i] for i in kidx]
        self.prog.accs = [ir.Acc(kind, s, bits) for (kind, _, bits), s in zip(accs, slots[len(keys):])]
        return self.prog

    def _lower_aggregate(self, agg_func, combine_func, init):
        """Recognise component-wise `a (+) g(x)` aggregators with a matching associative combiner."""
        inits = list(init) if isinstance(init, (tuple, list)) else [init]
        n = len(inits)
        an, abody, aenv = get_udf_ast(agg_func)
        cn, cbody, _ = get_udf_ast(combine_func)
        if len(an) != 2 or len(cn) != 2:
            raise UnsupportedUDF("aggregate UDFs take (aggregate, row) and (a, b)")
        abody = _single_return(abody)
        cbody = _single_return(cbody)
        aparts = abody.elts if isinstance(abody, ast.Tuple) else [abody]
        cparts = cbody.elts if isinstance(cbody, ast.Tuple) else [cbody]
        if len(aparts) != n or len(cparts) != n:
            raise UnsupportedUDF("aggregate shape does not match initial value")

        def is_acc_ref(node, name, i):
            if n == 1 and isinstance(node, ast.Name) and node.id == name:
                return True
            return (isinstance(node, ast.Subscript) and isinstance(node.value, ast.Name) and node.value.id == name
                    and isinstance(node.slice, ast.Constant) and node.slice.value == i)

        out = []
        fc = _FuncCompiler(self, aenv)
        fc.env[an[1]] = self.row_value()
        for i, (ap, cp, iv) in enumerate(zip(aparts, cparts, inits)):
            kind = None
            g_node = None
            if isinstance(ap, ast.BinOp) and isinstance(ap.op, ast.Add):
                if is_acc_ref(ap.left, an[0], i):
                    g_node, kind = ap.right, "sum"
                elif is_acc_ref(ap.right, an[0], i):
                    g_node, kind = ap.left, "sum"
            elif isinstance(ap, ast.Call) and isinstance(ap.func, ast.Name) and ap.func.id in ("min", "max") and len(ap.args) == 2:
                if is_acc_ref(ap.args[0], an[0], i):
                    g_node, kind = ap.args[1], ap.func.id
                elif is_acc_ref(ap.args[1], an[0], i):
                    g_node, kind = ap.args[0], ap.func.id
            if kind is None or _mentions(g_node, an[0]):
                raise UnsupportedUDF("aggregate component is not of the form a (+) g(x)")
            # combiner must be the same associative operation on component i
            ok = False
            if kind == "sum" and isinstance(cp, ast.BinOp) and isinstance(cp.op, ast.Add):
                ok = (is_acc_ref(cp.left, cn[0], i) and is_acc_ref(cp.right, cn[1], i)) or \
                     (is_acc_ref(cp.left, cn[1], i) and is_acc_ref(cp.right, cn[0], i))
            elif kind in ("min", "max") and isinstance(cp, ast.Call) and isinstance(cp.func, ast.Name) and cp.func.id == kind and len(cp.args) == 2:
                ok = {0, 1} == {j for j in (0, 1) for a_ in cp.args if is_acc_ref(a_, cn[j], i)}
            if not ok:
                raise UnsupportedUDF("combine UDF does not match the aggregate operation")
            g = fc.expr(g_node)
            if isinstance(g, TupleVal) or g.type == T_STR:
                raise UnsupportedUDF("aggregate term must be numeric")
            if isinstance(iv, bool) or not isinstance(iv, (int, float)):
                raise UnsupportedUDF("initial aggregate value must be int or float")
            is_f = g.type == T_F64 or isinstance(iv, float)
            if is_f:
                g = self.to_f64(g)
                bits = ir.f64_bits(float(iv))
                k = {"sum": "TPLX_ACC_SUM_F64", "min": "TPLX_ACC_MIN_F64", "max": "TPLX_ACC_MAX_F64"}[kind]
            else:
                g = self.to_i64(g)
                bits = int(iv) & ((1 << 64) - 1)
                k = {"sum": "TPLX_ACC_SUM_I64", "min": "TPLX_ACC_MIN_I64", "max": "TPLX_ACC_MAX_I64"}[kind]
            out.append((C[k], g, bits))
        return out

    # ---- register allocation -----------------------------------------------------------------------
    def _regalloc(self, live_out: List[int]) -> List[int]:
        """Linear-scan assignment of vregs to 8-byte slots (strings take two consecutive slots).
        The program is straight-line (predicated), so a vreg's live range is [first def, last use]."""
        ins = self.prog.instrs
        n = len(self.vreg_width)
        first = [None] * n
        last = [-1] * n
        for pc, i in enumerate(ins):
            for r in (i.a, i.b, i.c, i.guard):
                if r != NOSLOT:
                    last[r] = max(last[r], pc)
                    if first[r] is None:
                        first[r] = pc  # used before def can only be a guarded phi input; treat as live from here
            if i.dst != NOSLOT:
                if first[i.dst] is None:
                    first[i.dst] = pc
                last[i.dst] = max(last[i.dst], pc)
        for r in live_out:
            last[r] = len(ins)
        # a vreg that is redefined under guards (phi via repeated MOV) stays live across all its defs: covered by min/max
        order = sorted((r for r in range(n) if first[r] is not None), key=lambda r: first[r])
        free1: List[int] = []
        free2: List[int] = []
        active: List[Tuple[int, int]] = []  # (end, vreg)
        assign: Dict[int, int] = {}
        top = 0
        for r in order:
            start = first[r]
            still = []
            for end, v in active:
                if end < start:
                    (free2 if self.vreg_width[v] == 2 else free1).append(assign[v])
                else:
                    still.append((end, v))
            active = still
            w = self.vreg_width[r]
            if w == 2:
                if free2:
                    s = free2.pop()
                else:
                    s = top
                    top += 2
            else:
                if free1:
                    s = free1.pop()
                elif free2:
                    s = free2.pop()
                    free1.append(s + 1)
                else:
                    s = top
                    top += 1
            assign[r] = s
            active.append((last[r], r))
        for i in ins:
            for f in ("dst", "a", "b", "c", "guard"):
                v = getattr(i, f)
                if v != NOSLOT:
                    setattr(i, f, assign[v])
        self.prog.n_slots = max(top, 1)
        if self.prog.n_slots >= NOSLOT:
            raise UnsupportedUDF("program too large")
        return [assign[r] for r in live_out]


def _match_string_scan(sc: "StageCompiler") -> Optional[bytes]:
    """Recognise a row-index stage (the prefilter of a selective pipeline) that is nothing but a chain of filters of the closed
    forms of include/tplx_ir.h (tplx_scan_term: CONTAINS / FIELD_INT / FIXED) and state it as a string-scan hint. Works on the
    vreg program after dead-code elimination and idiom fusion; every instruction has to be explained by a term, otherwise None."""
    OP = lambda k: C["TPLX_OP_" + k]
    AC, BC, CC = C["TPLX_F_A_CONST"], C["TPLX_F_B_CONST"], C["TPLX_F_C_CONST"]
    sym: Dict[int, tuple] = {}
    terms: List[dict] = []
    ins = sc.prog.instrs
    mirror = {C["TPLX_CMP_LT"]: C["TPLX_CMP_GT"], C["TPLX_CMP_GT"]: C["TPLX_CMP_LT"], C["TPLX_CMP_LE"]: C["TPLX_CMP_GE"],
              C["TPLX_CMP_GE"]: C["TPLX_CMP_LE"], C["TPLX_CMP_EQ"]: C["TPLX_CMP_EQ"], C["TPLX_CMP_NE"]: C["TPLX_CMP_NE"]}
    for pc, i in enumerate(ins):
        if i.guard != NOSLOT:
            return None
        a, b, c_ = sym.get(i.a), sym.get(i.b), sym.get(i.c)
        fl = i.flags
        if i.op == OP("LDCOL"):
            sym[i.dst] = ("col", int(i.imm), i.flags, 0)
        elif i.op in (OP("SLOWER"), OP("SUPPER")) and a and a[0] == "col" and a[2] == T_STR and a[3] == 0 and not (fl & AC):
            sym[i.dst] = ("col", a[1], T_STR, C["TPLX_SF_LOWER"] if i.op == OP("SLOWER") else C["TPLX_SF_UPPER"])
        elif i.op == OP("SFINDE") and a and a[0] == "col" and a[2] == T_STR and a[3] == 0 and (fl & BC) and not (fl & AC):
            sym[i.dst] = ("finde", a[1], int(i.imm))
        elif (i.op == OP("SSLICE") and a and a[0] == "col" and a[2] == T_STR and a[3] == 0 and (fl & 3) == C["TPLX_SL_HAS_END"]
              and not (fl & (AC | BC | CC)) and c_ and c_[0] == "finde" and c_[1] == a[1]):
            sym[i.dst] = ("head", a[1], c_[2])
        elif i.op == OP("SRFINDK") and a and a[0] == "head" and (fl & BC):
            sym[i.dst] = ("rfk", a[1], a[2], int(i.imm), int(i.imm2))
        elif (i.op == OP("SSLICE") and a and a[0] == "head" and (fl & 3) == C["TPLX_SL_HAS_START"] and not (fl & (AC | BC | CC))
              and b and b[0] == "rfk" and b[1:3] == a[1:3]):
            sym[i.dst] = ("field", a[1], a[2], b[3], b[4])
        elif i.op == OP("S2I") and a and a[0] == "field" and not (fl & AC):
            sym[i.dst] = ("fieldint",) + a[1:] + (i.opidx,)
        elif i.op == OP("ICMP") and (fl & (AC | BC)) in (AC, BC):
            v = b if (fl & AC) else a
            k = int(i.imm2 if (fl & AC) else i.imm)
            cmp_ = mirror[fl & 7] if (fl & AC) else (fl & 7)
            if v and v[0] == "fieldint":
                sym[i.dst] = ("pred", dict(kind=C["TPLX_SK_FIELD_INT"], col=v[1], flags=0, cmp=cmp_, imm=k, needle=v[2], sep=v[3], skip=v[4],
                                           opidx_val=v[5]))
            elif v and v[0] == "col" and v[2] in (T_I64, T_BOOL):
                sym[i.dst] = ("pred", dict(kind=C["TPLX_SK_FIXED"], col=v[1], flags=0, cmp=cmp_, imm=k))
            else:
                return None
        elif i.op == OP("FCMP") and (fl & (AC | BC)) in (AC, BC):
            v = b if (fl & AC) else a
            k = int(i.imm2 if (fl & AC) else i.imm)
            if not (v and v[0] == "col" and v[2] == T_F64):
                return None
            sym[i.dst] = ("pred", dict(kind=C["TPLX_SK_FIXED"], col=v[1], flags=C["TPLX_SCF_F64"], cmp=mirror[fl & 7] if (fl & AC) else (fl & 7), imm=k))
        elif i.op == OP("SIN") and (fl & AC) and not (fl & BC) and b and b[0] == "col" and b[2] == T_STR:
            sym[i.dst] = ("pred", dict(kind=C["TPLX_SK_CONTAINS"], col=b[1], flags=b[3], needle=int(i.imm2)))
        elif i.op == OP("BNOT") and a and a[0] == "pred" and a[1]["kind"] == C["TPLX_SK_CONTAINS"] and not (fl & AC):
            t = dict(a[1])
            t["flags"] ^= C["TPLX_SCF_NEGATE"]
            sym[i.dst] = ("pred", t)
        elif i.op == OP("FILTER") and a and a[0] == "pred":
            t = dict(a[1])
            t["opidx_filter"] = i.opidx
            terms.append(t)
        elif i.op == OP("LDROW") and pc == len(ins) - 1:
            pass
        else:
            return None
    if not terms or len(terms) > C["TPLX_MAX_SCAN_TERMS"]:
        return None
    # every value that can raise must feed a filter: an int() whose result nobody tests would be lost by the closed form
    n_field = sum(1 for i in ins if i.op == OP("S2I"))
    if n_field != sum(1 for t in terms if t["kind"] == C["TPLX_SK_FIELD_INT"]):
        return None
    return ir.pack_scan_terms(terms)


def _match_fused_scan_aggregate(sc: "StageCompiler", agg_func, combine_func, init) -> Optional[bytes]:
    """Recognise the closed form `filters of (column <op> constant) ranges -> sum of const | col | col*col`
    (include/tplx_ir.h tplx_fused_header). Returns the serialized hint or None. Works on a scratch compiler so the
    real program is untouched; constants go through the same folding (incl. the reference's 6-digit quirk)."""
    import struct
    if any(name != "add_filter" for name, _ in sc.oplog):
        return None
    tmp = StageCompiler(sc.prog.in_types, sc.prog.in_names)
    fixed = (T_I64, T_F64, T_BOOL)

    def col_of(v):
        if isinstance(v, Val) and tmp._is_colref(v) and v.type in fixed:
            return v.const[1]
        return None

    preds = {}  # col -> [flags, lo, hi] merged per column and compare domain

    def add_bound(col, as_f64, cast, is_lo, value, incl):
        key = (col, as_f64)
        e = preds.setdefault(key, {"lo": None, "hi": None, "cast": cast})
        cur = e["lo" if is_lo else "hi"]
        cand = (value, incl)
        if cur is None:
            e["lo" if is_lo else "hi"] = cand
        else:  # keep the tighter bound
            if is_lo:
                tighter = cand[0] > cur[0] or (cand[0] == cur[0] and not cand[1])
            else:
                tighter = cand[0] < cur[0] or (cand[0] == cur[0] and not cand[1])
            if tighter:
                e["lo" if is_lo else "hi"] = cand

    def one_compare(op, l, r):
        cl, cr = col_of(l), col_of(r)
        if (cl is None) == (cr is None):
            raise UnsupportedUDF("fused: need exactly one column per comparison")
        col = cl if cl is not None else cr
        k = r if cl is not None else l
        if not tmp.is_const(k) or isinstance(k.const, str):
            raise UnsupportedUDF("fused: non-constant bound")
        ctype = tmp.row[col].type
        as_f64 = ctype == T_F64 or isinstance(k.const, float)
        cast = as_f64 and ctype != T_F64
        val = float(k.const) if as_f64 else int(k.const)
        t = type(op)
        if cl is None:  # const OP col  ->  col OP' const
            t = {ast.Lt: ast.Gt, ast.LtE: ast.GtE, ast.Gt: ast.Lt, ast.GtE: ast.LtE, ast.Eq: ast.Eq}.get(t)
        if t is ast.Lt:
            add_bound(col, as_f64, cast, False, val, False)
        elif t is ast.LtE:
            add_bound(col, as_f64, cast, False, val, True)
        elif t is ast.Gt:
            add_bound(col, as_f64, cast, True, val, False)
        elif t is ast.GtE:
            add_bound(col, as_f64, cast, True, val, True)
        elif t is ast.Eq:
            add_bound(col, as_f64, cast, True, val, True)
            add_bound(col, as_f64, cast, False, val, True)
        else:
            raise UnsupportedUDF("fused: comparison operator")

    def walk(fc, node):
        if isinstance(node, ast.BoolOp) and isinstance(node.op, ast.And):
            for v in node.values:
                walk(fc, v)
            return
        if not isinstance(node, ast.Compare):
            raise UnsupportedUDF("fused: filter is not a comparison")
        left = fc.expr(node.left)
        for op, rn in zip(node.ops, node.comparators):
            right = fc.expr(rn)
            one_compare(op, left, right)
            left = right

    for _, (func, _opid) in sc.oplog:
        argn, body, env = get_udf_ast(func)
        body = _single_return(body)
        if len(argn) != 1:
            raise UnsupportedUDF("fused: filter arity")
        fc = _FuncCompiler(tmp, env)
        fc.env[argn[0]] = tmp.row_value()
        walk(fc, body)
    if len(tmp.prog.instrs):
        raise UnsupportedUDF("fused: filter needed run-time evaluation")

    # aggregate terms
    inits = list(init) if isinstance(init, (tuple, list)) else [init]
    an, abody, aenv = get_udf_ast(agg_func)
    abody = _single_return(abody)
    parts = abody.elts if isinstance(abody, ast.Tuple) else [abody]
    if len(an) != 2 or len(parts) != len(inits):
        raise UnsupportedUDF("fused: aggregate shape")
    terms = []
    fc = _FuncCompiler(tmp, aenv)
    fc.env[an[1]] = tmp.row_value()
    for i, (ap, iv) in enumerate(zip(parts, inits)):
        if not (isinstance(ap, ast.BinOp) and isinstance(ap.op, ast.Add)):
            raise UnsupportedUDF("fused: term")

        def is_acc(n_):
            if len(inits) == 1 and isinstance(n_, ast.Name) and n_.id == an[0]:
                return True
            return (isinstance(n_, ast.Subscript) and isinstance(n_.value, ast.Name) and n_.value.id == an[0]
                    and isinstance(n_.slice, ast.Constant) and n_.slice.value == i)
        g = ap.right if is_acc(ap.left) else ap.left if is_acc(ap.right) else None
        if g is None or _mentions(g, an[0]):
            raise UnsupportedUDF("fused: term")
        is_f = isinstance(iv, float)
        if isinstance(g, ast.BinOp) and isinstance(g.op, ast.Mult):
            a_, b_ = fc.expr(g.left), fc.expr(g.right)
            ca, cb = col_of(a_), col_of(b_)
            if ca is None or cb is None:
                raise UnsupportedUDF("fused: product of non-columns")
            ta, tb = tmp.row[ca].type, tmp.row[cb].type
            f = is_f or ta == T_F64 or tb == T_F64
            terms.append((C["TPLX_ACC_SUM_F64"] if f else C["TPLX_ACC_SUM_I64"], C["TPLX_FT_MUL"], ca, cb,
                          int(f and ta != T_F64), int(f and tb != T_F64), 0))
        else:
            v = fc.expr(g)
            cv = col_of(v)
            if cv is not None:
                f = is_f or tmp.row[cv].type == T_F64
                terms.append((C["TPLX_ACC_SUM_F64"] if f else C["TPLX_ACC_SUM_I64"], C["TPLX_FT_COL"], cv, 0,
                              int(f and tmp.row[cv].type != T_F64), 0, 0))
            elif tmp.is_const(v) and not isinstance(v.const, str):
                f = is_f or isinstance(v.const, float)
                imm = ir.f64_bits(float(v.const)) if f else int(v.const) & ((1 << 64) - 1)
                terms.append((C["TPLX_ACC_SUM_F64"] if f else C["TPLX_ACC_SUM_I64"], C["TPLX_FT_CONST"], 0, 0, 0, 0, imm))
            else:
                raise UnsupportedUDF("fused: term")
    if len(tmp.prog.instrs) or len(preds) > C["TPLX_MAX_FUSED_PREDS"] or not terms:
        raise UnsupportedUDF("fused: not closed form")
    # the combiner must be the matching sum (checked by _lower_aggregate on the real program)
    out = struct.pack("<IIII", C["TPLX_FUSED_MAGIC"], len(preds), len(terms), 0)
    for (col, as_f64), e in preds.items():
        fl = (C["TPLX_FP_F64"] if as_f64 else 0) | (C["TPLX_FP_CAST"] if e["cast"] else 0)
        lo = hi = 0
        if e["lo"] is not None:
            fl |= C["TPLX_FP_HAS_LO"] | (C["TPLX_FP_LO_INCL"] if e["lo"][1] else 0)
            lo = ir.f64_bits(e["lo"][0]) if as_f64 else e["lo"][0] & ((1 << 64) - 1)
        if e["hi"] is not None:
            fl |= C["TPLX_FP_HAS_HI"] | (C["TPLX_FP_HI_INCL"] if e["hi"][1] else 0)
            hi = ir.f64_bits(e["hi"][0]) if as_f64 else e["hi"][0] & ((1 << 64) - 1)
        out += struct.pack("<IIQQ", col, fl, lo, hi)
    for t in terms:
        out += struct.pack("<IIIIIIQ", *t)
    return out


def _single_return(body):
    if isinstance(body, list):
        stmts = [s for s in body if not (isinstance(s, ast.Expr) and isinstance(s.value, ast.Constant))]
        if len(stmts) == 1 and isinstance(stmts[0], ast.Return) and stmts[0].value is not None:
            return stmts[0].value
        raise UnsupportedUDF("aggregate UDF must be a single expression")
    return body


def _mentions(node, name) -> bool:
    return any(isinstance(n, ast.Name) and n.id == name for n in ast.walk(node))


# ------------------------------------------------------------------------------------------------
# per-function lowering
# ------------------------------------------------------------------------------------------------
_CMP = {ast.Eq: "EQ", ast.NotEq: "NE", ast.Lt: "LT", ast.LtE: "LE", ast.Gt: "GT", ast.GtE: "GE"}
_FMT_RE = re.compile(r"%(?:(?P<flags>[0 \-+#]*)(?P<width>\d*)(?:\.(?P<prec>\d+))?(?P<conv>[dsif%]))")


class _FuncCompiler:
    def __init__(self, sc: StageCompiler, genv: Dict[str, Any]):
        self.sc = sc
        self.genv = genv
        self.env: Dict[str, Any] = {}
        self.ret_val = None
        self.ret_done: Val = const_val(False)  # "row has already returned"
        self.path: Optional[Val] = None         # conjunction of enclosing if-conditions

    # guard management -------------------------------------------------------------------------------
    def _set_guard(self):
        g = self.path
        if not (self.sc.is_const(self.ret_done) and not self.ret_done.const):
            # the guard of the next statement is a value every row must have: computed outside any guard (an instruction that is
            # skipped leaves its destination undefined, and an undefined guard would let rows run or skip the statement at random)
            g = self._with_unguarded(lambda: self.sc.b_and(g, self.sc.b_not(self.ret_done)) if g is not None else self.sc.b_not(self.ret_done))
        if g is None:
            self.sc.guard = None
        elif self.sc.is_const(g):
            self.sc.guard = None if g.const else self.sc.reg(g)
        else:
            self.sc.guard = self.sc.reg(g)

    def _with_unguarded(self, fn):
        g = self.sc.guard
        self.sc.guard = None
        try:
            return fn()
        finally:
            self.sc.guard = g

    def run(self, argnames, args_vals, body):
        outer_guard = self.sc.guard
        for n, v in zip(argnames, args_vals):
            self.env[n] = v
        if isinstance(body, list):
            self.block(body)
            if self.ret_val is None:
                raise UnsupportedUDF("function does not return a value")
            res = self.ret_val
        else:
            self._set_guard()
            res = self.expr(body)
        self.sc.guard = outer_guard
        return res

    # statements -------------------------------------------------------------------------------------
    def block(self, stmts):
        for s in stmts:
            self._set_guard()
            self.stmt(s)

    def stmt(self, s):
        sc = self.sc
        if isinstance(s, ast.Return):
            if s.value is None:
                raise UnsupportedUDF("return without value")
            v = self.expr(s.value)
            here = self.path if self.path is not None else const_val(True)
            active = self._with_unguarded(lambda: sc.b_and(here, sc.b_not(self.ret_done)))
            if self.ret_val is None:
                self.ret_val = v
            else:
                self.ret_val = self._with_unguarded(lambda: sc.select(active, v, self.ret_val))
            self.ret_done = self._with_unguarded(lambda: sc.b_or(self.ret_done, here))
            return
        if isinstance(s, ast.Assign):
            if len(s.targets) != 1:
                raise UnsupportedUDF("chained assignment")
            v = self.expr(s.value)
            self._assign(s.targets[0], v)
            return
        if isinstance(s, ast.AugAssign):
            if not isinstance(s.target, ast.Name):
                raise UnsupportedUDF("augmented assignment target")
            cur = self.expr(ast.Name(id=s.target.id, ctx=ast.Load()))
            v = self.binop(s.op, cur, self.expr(s.value))
            self._assign(s.target, v)
            return
        if isinstance(s, ast.If):
            cond = sc.truth(self.expr(s.test))
            outer_path, outer_env = self.path, dict(self.env)
            # then-branch
            self.path = self._with_unguarded(lambda: sc.b_and(outer_path, cond) if outer_path is not None else cond)
            self.block(s.body)
            env_then = self.env
            # else-branch
            self.env = dict(outer_env)
            ncond = self._with_unguarded(lambda: sc.b_not(cond))
            self.path = self._with_unguarded(lambda: sc.b_and(outer_path, ncond) if outer_path is not None else ncond)
            self.block(s.orelse)
            env_else = self.env
            self.path = outer_path
            # merge variables
            merged = dict(outer_env)
            for name in set(env_then) | set(env_else):
                a, b = env_then.get(name), env_else.get(name)
                if a is b:
                    merged[name] = a
                elif a is None:
                    merged[name] = b
                elif b is None:
                    merged[name] = a
                else:
                    merged[name] = self._with_unguarded(lambda a=a, b=b: sc.select(cond, a, b))
            self.env = merged
            return
        if isinstance(s, ast.Expr):
            if isinstance(s.value, ast.Constant):
                return  # docstring
            self.expr(s.value)
            return
        if isinstance(s, ast.Pass):
            return
        raise UnsupportedUDF(f"statement {type(s).__name__} not supported")

    def _assign(self, target, v):
        if isinstance(target, ast.Name):
            self.env[target.id] = v
            return
        if isinstance(target, ast.Tuple) and isinstance(v, TupleVal) and len(target.elts) == len(v.elems):
            for t, e in zip(target.elts, v.elems):
                self._assign(t, e)
            return
        raise UnsupportedUDF("assignment target not supported")

    # expressions ------------------------------------------------------------------------------------
    def expr(self, e):
        sc = self.sc
        if isinstance(e, ast.Constant):
            if e.value is None:
                return none_val()
            return const_val(e.value)
        if isinstance(e, ast.Name):
            if e.id in self.env:
                return self.env[e.id]
            if e.id in ("True", "False"):
                return const_val(e.id == "True")
            if e.id in self.genv and isinstance(self.genv[e.id], (bool, int, float, str)):
                return const_val(self.genv[e.id])
            raise UnsupportedUDF(f"name {e.id!r} is not a parameter, local or constant global")
        if isinstance(e, ast.Tuple):
            return TupleVal([self.expr(x) for x in e.elts])
        if isinstance(e, ast.List):
            tv = TupleVal([self.expr(x) for x in e.elts])
            tv.is_list = True  # only usable as the container of an `in` test; a list-valued column is not normal-case
            return tv
        if isinstance(e, ast.Dict):
            # {'a': e1, 'b': e2}: a row with named columns (python/tuplex/dataset.py map() with dict output)
            if not all(isinstance(k, ast.Constant) and isinstance(k.value, str) for k in e.keys):
                raise UnsupportedUDF("dict keys must be string literals")
            return TupleVal([self.expr(v) for v in e.values], [k.value for k in e.keys])
        if isinstance(e, ast.JoinedStr):
            return self.format_pieces([("lit", p.value) if isinstance(p, ast.Constant) else
                                       ("val", self.need(self.expr(p.value)), self._spec_of(p)) for p in e.values])
        if isinstance(e, ast.BinOp):
            return self.binop(e.op, self.expr(e.left), self.expr(e.right))
        if isinstance(e, ast.UnaryOp):
            v = self.expr(e.operand)
            if isinstance(e.op, ast.Not):
                return sc.b_not(sc.truth(v))
            v = self.need(v)
            if isinstance(v, TupleVal) or v.type == T_STR:
                raise UnsupportedUDF("unary operator on non-number")
            if isinstance(e.op, ast.USub):
                if sc.is_const(v):
                    return const_val(-v.const if not isinstance(v.const, bool) else -int(v.const))
                return sc.op1(C["TPLX_OP_FNEG"], T_F64, v) if v.type == T_F64 else sc.op1(C["TPLX_OP_INEG"], T_I64, sc.to_i64(v))
            if isinstance(e.op, ast.UAdd):
                return v if v.type == T_F64 else sc.to_i64(v)
            if isinstance(e.op, ast.Invert):
                return sc.op2(C["TPLX_OP_IXOR"], T_I64, sc.to_i64(v), const_val(-1))
        if isinstance(e, ast.BoolOp):
            # short-circuit: later operands are only evaluated (and may only raise) when needed
            vals = None
            outer_path = self.path
            acc = None
            for i, sub in enumerate(e.values):
                v = sc.truth(self.expr(sub))
                if acc is None:
                    acc = v
                else:
                    acc = self._with_unguarded(lambda: sc.b_and(acc, v)) if isinstance(e.op, ast.And) else \
                        self._with_unguarded(lambda: sc.b_or(acc, v))
                if i + 1 < len(e.values):
                    need = acc if isinstance(e.op, ast.And) else self._with_unguarded(lambda: sc.b_not(acc))
                    self.path = self._with_unguarded(lambda: sc.b_and(outer_path, need) if outer_path is not None else need)
                    self._set_guard()
            self.path = outer_path
            self._set_guard()
            return acc
        if isinstance(e, ast.Compare):
            return self.compare(e)
        if isinstance(e, ast.IfExp):
            cond = sc.truth(self.expr(e.test))
            outer_path = self.path
            self.path = self._with_unguarded(lambda: sc.b_and(outer_path, cond) if outer_path is not None else cond)
            self._set_guard()
            a = self.expr(e.body)
            ncond = self._with_unguarded(lambda: sc.b_not(cond))
            self.path = self._with_unguarded(lambda: sc.b_and(outer_path, ncond) if outer_path is not None else ncond)
            self._set_guard()
            b = self.expr(e.orelse)
            self.path = outer_path
            self._set_guard()
            return sc.select(cond, a, b)
        if isinstance(e, ast.Subscript):
            return self.subscript(e)
        if isinstance(e, ast.Call):
            return self.call(e)
        raise UnsupportedUDF(f"expression {type(e).__name__} not supported")

    # ---- arithmetic (BlockGeneratorVisitor.cc:152-584) ------------------------------------------------
    def binop(self, op, l, r):
        sc = self.sc
        if isinstance(l, TupleVal) or isinstance(r, TupleVal):
            raise UnsupportedUDF("tuple arithmetic")
        l, r = self.need(l), self.need(r)
        if l.type == T_STR or r.type == T_STR:
            if isinstance(op, ast.Add) and l.type == T_STR and r.type == T_STR:
                if sc.is_const(l) and sc.is_const(r):
                    return const_val(l.const + r.const)
                return sc.op2(C["TPLX_OP_SCONCAT"], T_STR, l, r)
            if isinstance(op, ast.Mod) and l.type == T_STR:
                return self.format_percent(l, r)
            raise UnsupportedUDF("string operator not supported")
        if isinstance(op, ast.Pow):
            return self.power(self._force(l) if sc.is_const(l) else l, r)
        if sc.is_const(l) and sc.is_const(r):
            return self.fold(op, l.const, r.const)
        is_f = l.type == T_F64 or r.type == T_F64
        if isinstance(op, ast.Div):
            return sc.op2(C["TPLX_OP_FDIV"], T_F64, sc.to_f64(l), sc.to_f64(r))
        if is_f:
            table = {ast.Add: "FADD", ast.Sub: "FSUB", ast.Mult: "FMUL", ast.Mod: "FMOD", ast.FloorDiv: "FFLOORDIV"}
            if type(op) not in table:
                raise UnsupportedUDF(f"float operator {type(op).__name__}")
            return sc.op2(C["TPLX_OP_" + table[type(op)]], T_F64, sc.to_f64(l), sc.to_f64(r))
        table = {ast.Add: "IADD", ast.Sub: "ISUB", ast.Mult: "IMUL", ast.Mod: "IMOD", ast.FloorDiv: "IFLOORDIV",
                 ast.BitAnd: "IAND", ast.BitOr: "IOR", ast.BitXor: "IXOR", ast.LShift: "ISHL", ast.RShift: "ISHR"}
        if type(op) not in table:
            raise UnsupportedUDF(f"integer operator {type(op).__name__}")
        if type(op) in (ast.BitAnd, ast.BitOr, ast.BitXor) and l.type == T_BOOL and r.type == T_BOOL:
            return sc.op2(C["TPLX_OP_" + table[type(op)]], T_BOOL, l, r)
        return sc.op2(C["TPLX_OP_" + table[type(op)]], T_I64, sc.to_i64(l), sc.to_i64(r))

    def power(self, l: Val, r: Val) -> Val:
        """base ** k for a literal integer exponent |k| <= 6: the reference's constant-exponent code
        (BlockGeneratorVisitor::powerInst :1313-1522 -> generateConstantIntegerPower :5837-5957): addition chains of single
        multiplies (wrapping i64 / IEEE f64, same association), base == 0 short-cuts to 0, a negative exponent gives
        1.0 / power as f64 and ZeroDivisionError for base == 0. Other exponents (its general path speculates on the sign of
        the exponent and calls libm pow; its chain for |k| >= 7 is not a power) stay on the CPython path."""
        sc = self.sc
        if not (sc.is_const(r) and r.type in (T_I64, T_BOOL)) or l.type == T_STR:
            raise UnsupportedUDF("** needs a literal integer exponent")
        k = int(r.const)
        if abs(k) > 6:
            raise UnsupportedUDF("** with |exponent| > 6")
        base = sc.to_f64(l) if l.type == T_F64 else sc.to_i64(l)
        is_f = base.type == T_F64
        if k == 0:
            return const_val(1.0 if is_f else 1)
        zero = const_val(0.0 if is_f else 0)
        is_zero = sc.op2(C["TPLX_OP_FCMP" if is_f else "TPLX_OP_ICMP"], T_BOOL, base, zero, flags=C["TPLX_CMP_EQ"])
        if k < 0:
            self.raise_if(is_zero, C["TPLX_EC_ZERODIVISIONERROR"])
        mul = lambda a, b: sc.op2(C["TPLX_OP_FMUL" if is_f else "TPLX_OP_IMUL"], base.type, a, b)
        n = abs(k)
        if n == 1:
            p = base
        else:
            b2 = mul(base, base)
            if n == 2:
                p = b2
            elif n == 3:
                p = mul(b2, base)
            else:
                b4 = mul(b2, b2)
                p = b4 if n == 4 else (mul(base, b4) if n == 5 else mul(b2, b4))
        if k < 0:
            return sc.op2(C["TPLX_OP_FDIV"], T_F64, const_val(1.0), p if is_f else sc.to_f64(p))
        # base == 0 -> the constant 0 / 0.0 (for -0.0 too: FCmpOEQ(-0.0, 0.0) holds)
        return sc.select(is_zero, zero, p) if is_f else p

    def need(self, v):
        """A value about to be USED (arithmetic, call argument, index ...): for an Option[T] value the rows that hold None raise
        TypeError here — on the executed path only, like every exception (PipelineBuilder.cc:949) — and take the interpreter path,
        where CPython decides what `None + 1` or `str(None)` means; the other rows go on with the plain T value."""
        if isinstance(v, TupleVal) or v.null is None:
            return v
        if v.type == T_NONE:
            raise UnsupportedUDF("the literal None used as a value")
        self.raise_if(v.null, C["TPLX_EC_TYPEERROR"])
        return plain(v)

    def raise_if(self, cond: Val, code: int):
        """Raise `code` for the rows where cond holds (on the executed path only)."""
        sc = self.sc
        if sc.is_const(cond) and not cond.const:
            return
        g = sc.guard
        if sc.is_const(cond):
            sc.emit(C["TPLX_OP_RAISE"], imm=code)
            return
        both = cond if g is None else self._with_unguarded(lambda: sc.b_and(Val(T_BOOL, g), cond))
        sc.guard = sc.reg(both)
        sc.emit(C["TPLX_OP_RAISE"], imm=code)
        sc.guard = g

    def fold(self, op, a, b):
        """Literal folding with the reference's quirk: folded floats are re-parsed from their
        6-significant-digit text (ReduceExpressionsVisitor.cc:257-263,300-306,328-334)."""
        try:
            if isinstance(op, ast.Add):
                x = a + b
            elif isinstance(op, ast.Sub):
                x = a - b
            elif isinstance(op, ast.Mult):
                x = a * b
            elif isinstance(op, ast.Div):
                x = a / b
            else:
                # not folded by the reference: evaluate at run time so that errors surface per row
                return self.binop(op, self._force(const_val(a)), self._force(const_val(b)))
        except ZeroDivisionError:
            return self.binop(op, self._force(const_val(a)), self._force(const_val(b)))
        if isinstance(x, float):
            x = float("%g" % x)
        elif isinstance(x, bool):
            x = int(x)
        return const_val(x)

    def _force(self, v: Val) -> Val:
        return Val(v.type, self.sc.reg(v))

    def format_percent(self, fmt: Val, arg):
        """'%05d' % v via snprintf semantics (BlockGeneratorVisitor::formatStr :675-775)."""
        sc = self.sc
        if not sc.is_const(fmt):
            raise UnsupportedUDF("format string must be a literal")
        args = arg.elems if isinstance(arg, TupleVal) else [arg]
        pieces: List[Val] = []
        pos = 0
        ai = 0
        s = fmt.const
        for m in _FMT_RE.finditer(s):
            if m.start() > pos:
                pieces.append(const_val(s[pos:m.start()]))
            pos = m.end()
            conv = m.group("conv")
            if conv == "%":
                pieces.append(const_val("%"))
                continue
            if ai >= len(args):
                raise UnsupportedUDF("not enough arguments for format string")
            a = args[ai]
            ai += 1
            flags, width = m.group("flags") or "", int(m.group("width") or 0)
            if m.group("prec") or any(f in flags for f in " -+#"):
                raise UnsupportedUDF("format flags/precision not supported")
            if conv in "di":
                if isinstance(a, TupleVal) or a.type not in (T_I64, T_BOOL):
                    raise UnsupportedUDF("%d needs an integer")
                pieces.append(sc.op1(C["TPLX_OP_SFMTD"], T_STR, sc.to_i64(a), flags=1 if "0" in flags else 0, imm=width))
            elif conv == "s":
                if isinstance(a, TupleVal) or a.type != T_STR or width:
                    raise UnsupportedUDF("%s supports plain strings only")
                pieces.append(a)
            else:
                raise UnsupportedUDF("%f formatting not supported")
        if ai != len(args):
            raise UnsupportedUDF("too many arguments for format string")
        if pos < len(s):
            pieces.append(const_val(s[pos:]))
        if not pieces:
            return const_val("")
        out = pieces[0]
        for p in pieces[1:]:
            out = self.binop(ast.Add(), out, p)
        return out

    # ---- '{}'.format(...) and f-strings (FunctionRegistry::createFormatCall -> strFormat, Runtime.cc:544-607) ------
    _BRACE = re.compile(r"\{\{|\}\}|\{(\d*)(?::([^{}]*))?\}")

    def _spec_of(self, fv: ast.FormattedValue) -> str:
        if fv.conversion not in (-1, 115):
            raise UnsupportedUDF("f-string conversion")
        if fv.format_spec is None:
            return ""
        if len(fv.format_spec.values) == 1 and isinstance(fv.format_spec.values[0], ast.Constant):
            return str(fv.format_spec.values[0].value)
        raise UnsupportedUDF("dynamic format spec")

    def format_braces(self, fmt: str, args):
        pieces = []
        pos = 0
        auto = 0
        for m in self._BRACE.finditer(fmt):
            if m.start() > pos:
                pieces.append(("lit", fmt[pos:m.start()]))
            pos = m.end()
            if m.group(0) in ("{{", "}}"):
                pieces.append(("lit", m.group(0)[0]))
                continue
            idx = int(m.group(1)) if m.group(1) else auto
            auto += 1
            if idx >= len(args):
                raise UnsupportedUDF("format() argument index")
            pieces.append(("val", args[idx], m.group(2) or ""))
        if pos < len(fmt):
            pieces.append(("lit", fmt[pos:]))
        return self.format_pieces(pieces)

    def format_pieces(self, pieces):
        sc = self.sc
        out = None
        for p in pieces:
            if p[0] == "lit":
                v = const_val(p[1])
            else:
                a, spec = p[1], p[2]
                if isinstance(a, TupleVal):
                    raise UnsupportedUDF("format of a tuple")
                if a.type == T_STR:
                    if spec not in ("", "s"):
                        raise UnsupportedUDF("string format spec")
                    v = a
                elif a.type in (T_I64,):
                    ms = re.fullmatch(r"(0?)(\d*)d?", spec)
                    if not ms:
                        raise UnsupportedUDF("integer format spec")
                    width = int(ms.group(2) or 0)
                    if sc.is_const(a):
                        v = const_val(format(a.const, spec))
                    elif width == 0:
                        v = sc.op1(C["TPLX_OP_I2S"], T_STR, a)
                    else:  # flags: bit0 zero pad, bit1 full 64-bit value (fmt / str.format, unlike C's %d)
                        v = sc.op1(C["TPLX_OP_SFMTD"], T_STR, a, flags=(1 if ms.group(1) else 0) | 2, imm=width)
                else:
                    raise UnsupportedUDF("format of float/bool")
            out = v if out is None else self.binop(ast.Add(), out, v)
        return out if out is not None else const_val("")

    # ---- comparisons (BlockGeneratorVisitor.cc:776-880) -------------------------------------------------
    def compare(self, e: ast.Compare):
        sc = self.sc
        left = self.expr(e.left)
        acc = None
        outer_path = self.path
        for k, (op, rn) in enumerate(zip(e.ops, e.comparators)):
            right = self.expr(rn)
            c = self.compare1(op, left, right)
            acc = c if acc is None else self._with_unguarded(lambda: sc.b_and(acc, c))
            left = right
            if k + 1 < len(e.ops):  # chained comparison short-circuits like `and`
                self.path = self._with_unguarded(lambda: sc.b_and(outer_path, acc) if outer_path is not None else acc)
                self._set_guard()
        self.path = outer_path
        self._set_guard()
        return acc

    def compare1(self, op, l, r):
        sc = self.sc
        if isinstance(op, (ast.In, ast.NotIn)) and isinstance(r, TupleVal):
            # x in (c1, c2, ...): membership in a literal tuple/list = a chain of equality tests
            if isinstance(l, TupleVal) or not r.elems:
                raise UnsupportedUDF("`in` over this container")
            acc = None
            for e_ in r.elems:
                c = self.compare1(ast.Eq(), l, e_)
                acc = c if acc is None else sc.b_or(acc, c)
            return sc.b_not(acc) if isinstance(op, ast.NotIn) else acc
        if isinstance(l, TupleVal) or isinstance(r, TupleVal):
            raise UnsupportedUDF("tuple comparison")
        if l.null is not None or r.null is not None:
            if isinstance(op, (ast.Eq, ast.NotEq, ast.Is, ast.IsNot)):
                return self.compare_option(op, l, r)
            l, r = self.need(l), self.need(r)  # ordering / containment with None: TypeError for those rows
        elif isinstance(op, (ast.Is, ast.IsNot)):
            raise UnsupportedUDF("`is` between values that are never None")
        if isinstance(op, (ast.In, ast.NotIn)):
            if l.type != T_STR or r.type != T_STR:
                raise UnsupportedUDF("`in` is supported for str in str")
            if sc.is_const(l) and sc.is_const(r):
                res = const_val(l.const in r.const)
            else:
                res = sc.op2(C["TPLX_OP_SIN"], T_BOOL, l, r)
            return sc.b_not(res) if isinstance(op, ast.NotIn) else res
        if type(op) not in _CMP:
            raise UnsupportedUDF(f"comparison {type(op).__name__}")
        if l.type == T_STR or r.type == T_STR:
            if l.type != r.type:
                # str == number is False in Python; the reference rejects it at compile time
                raise UnsupportedUDF("comparison between str and number")
            if not isinstance(op, (ast.Eq, ast.NotEq)):
                raise UnsupportedUDF("ordering comparison of strings")
            if sc.is_const(l) and sc.is_const(r):
                return const_val((l.const == r.const) == isinstance(op, ast.Eq))
            if sc.is_const(l) or sc.is_const(r):
                k, v = (l, r) if sc.is_const(l) else (r, l)
                folded = self._fold_eq_through_select(v, k.const)
                if folded is not None:
                    return folded if isinstance(op, ast.Eq) else sc.b_not(folded)
            return sc.op2(C["TPLX_OP_SEQ"], T_BOOL, l, r, flags=0 if isinstance(op, ast.Eq) else 1)
        pred = C["TPLX_CMP_" + _CMP[type(op)]]
        if sc.is_const(l) and sc.is_const(r):
            a, b = l.const, r.const
            return const_val({"EQ": a == b, "NE": a != b, "LT": a < b, "LE": a <= b, "GT": a > b, "GE": a >= b}[_CMP[type(op)]])
        if l.type == T_F64 or r.type == T_F64:
            return sc.op2(C["TPLX_OP_FCMP"], T_BOOL, sc.to_f64(l), sc.to_f64(r), flags=pred)
        return sc.op2(C["TPLX_OP_ICMP"], T_BOOL, sc.to_i64(l), sc.to_i64(r), flags=pred)

    def compare_option(self, op, l: Val, r: Val):
        """== / != / is / is not with Option[T] or None operands (BlockGeneratorVisitor.cc:1030-1150): None equals only None; two
        present values compare as their base types; no row raises."""
        sc = self.sc
        eq = isinstance(op, (ast.Eq, ast.Is))
        ln = l.null if l.null is not None else const_val(False)
        rn = r.null if r.null is not None else const_val(False)
        if l.type == T_NONE or r.type == T_NONE:
            res = sc.b_and(ln, rn) if (l.type == T_NONE and r.type == T_NONE) else (rn if l.type == T_NONE else ln)
            # `x is None`: true exactly for the None rows of x (the other side is None for every row)
            return res if eq else sc.b_not(res)
        if isinstance(op, (ast.Is, ast.IsNot)):
            raise UnsupportedUDF("`is` between two values")
        both_null = sc.b_and(ln, rn)
        any_null = sc.b_or(ln, rn)
        same = self.compare1(ast.Eq(), plain(l), plain(r))  # compares never raise: evaluated for every row, used where both are present
        res = sc.b_or(both_null, sc.b_and(sc.b_not(any_null), same))
        return res if eq else sc.b_not(res)

    def _fold_eq_through_select(self, v, k: str):
        """(cond ? 'a' : 'b') == 'k'  ->  logic over cond when every leaf is a constant (else None)."""
        sc = self.sc
        if sc.is_const(v):
            return const_val(v.const == k)
        if getattr(v, "sel", None) is None:
            return None
        cond, a, b = v.sel
        ea, eb = self._fold_eq_through_select(a, k), self._fold_eq_through_select(b, k)
        if ea is None or eb is None:
            return None
        return sc.select(cond, ea, eb)

    # ---- subscripts -------------------------------------------------------------------------------------
    def subscript(self, e: ast.Subscript):
        sc = self.sc
        base = self.expr(e.value)
        if isinstance(base, TupleVal):
            if isinstance(e.slice, ast.Slice):
                raise UnsupportedUDF("tuple slices")
            idx = self.expr(e.slice)
            if not sc.is_const(idx):
                raise UnsupportedUDF("tuple index must be a compile-time constant")
            k = idx.const
            if isinstance(k, str):
                if not base.names or k not in base.names:
                    raise UnsupportedUDF(f"unknown column {k!r}")
                return base.elems[base.names.index(k)]
            if isinstance(k, bool) or not isinstance(k, int) or not -len(base.elems) <= k < len(base.elems):
                raise UnsupportedUDF("tuple index out of range")
            return base.elems[k]
        if base.type != T_STR:
            # single-column rows: x[0] / x['col'] address the only column (python/tuplex/dataset.py semantics)
            if isinstance(e.slice, ast.Constant) and (e.slice.value == 0 or (isinstance(e.slice.value, str) and e.slice.value in sc.names)):
                return base
            raise UnsupportedUDF("subscript on a number")
        if isinstance(e.slice, ast.Slice):
            sl = e.slice
            if sl.step is not None:
                st = self.expr(sl.step)
                if not (sc.is_const(st) and st.const == 1):
                    raise UnsupportedUDF("slice stride other than 1")
            lo = self.need(self.expr(sl.lower)) if sl.lower is not None else None
            hi = self.need(self.expr(sl.upper)) if sl.upper is not None else None
            for v in (lo, hi):
                if v is not None and (isinstance(v, TupleVal) or v.type not in (T_I64, T_BOOL)):
                    raise UnsupportedUDF("slice bounds must be integers")
            if sc.is_const(base) and (lo is None or sc.is_const(lo)) and (hi is None or sc.is_const(hi)):
                return const_val(base.const[(lo.const if lo else None):(hi.const if hi else None)])
            flags = (C["TPLX_SL_HAS_START"] if lo is not None else 0) | (C["TPLX_SL_HAS_END"] if hi is not None else 0)
            d = sc.new_vreg(T_STR)
            sc.emit_vals(C["TPLX_OP_SSLICE"], d, base, sc.to_i64(lo) if lo is not None else None,
                         sc.to_i64(hi) if hi is not None else None, flags=flags)
            return Val(T_STR, d)
        idx = self.need(self.expr(e.slice))
        if isinstance(idx, TupleVal) or idx.type not in (T_I64, T_BOOL):
            # single string column addressed by name
            if sc.is_const(idx) and isinstance(idx.const, str) and idx.const in sc.names and len(sc.row) == 1:
                return base
            raise UnsupportedUDF("string index must be an integer")
        return sc.op2(C["TPLX_OP_SINDEX"], T_STR, base, sc.to_i64(idx))

    # ---- calls (FunctionRegistry.cc) --------------------------------------------------------------------
    def call(self, e: ast.Call):
        sc = self.sc
        if e.keywords:
            raise UnsupportedUDF("keyword arguments")
        if isinstance(e.func, ast.Name):
            name = e.func.id
            args = [self.expr(a) for a in e.args]
            if name != "bool":  # bool(None) is False; every other builtin raises TypeError on None
                args = [self.need(a) for a in args]
            if any(isinstance(a, TupleVal) for a in args):
                if name == "len" and len(args) == 1:
                    return const_val(len(args[0].elems))
                raise UnsupportedUDF("tuple argument")
            if name == "int":
                if not args:
                    return const_val(0)
                (a,) = args
                if a.type in (T_I64, T_BOOL):
                    return sc.to_i64(a)
                if a.type == T_F64:
                    return const_val(int(a.const)) if sc.is_const(a) else sc.op1(C["TPLX_OP_F2I"], T_I64, a)
                return sc.op1(C["TPLX_OP_S2I"], T_I64, a)
            if name == "float" and len(args) == 1 and args[0].type != T_STR:
                return sc.to_f64(args[0])
            if name == "float" and len(args) == 1 and not sc.is_const(args[0]):
                return sc.op1(C["TPLX_OP_S2F"], T_F64, args[0])  # fast_atod semantics (FunctionRegistry.cc createFloatCast)
            if name == "bool" and len(args) == 1:
                a = args[0]
                if isinstance(a, Val) and a.type == T_F64 and not sc.is_const(a):
                    # bool(f64) is NOT the truth test of `if x:`: createBoolCast compares with FCMP_OEQ and negates (FunctionRegistry.cc:396-399),
                    # so bool(nan) is True like in Python, while `if nan:` is false in the reference (truthValueTest, FCMP_ONE,
                    # LLVMEnvironment.cc:922-927; gtest golden UseCaseFunctionsTest.cc:183-197)
                    v = sc.b_not(sc.op2(C["TPLX_OP_FCMP"], T_BOOL, plain(a), const_val(0.0), flags=C["TPLX_CMP_EQ"]))
                    return v if a.null is None else sc.b_and(sc.b_not(a.null), v)
                return sc.truth(a)
            if name == "len" and len(args) == 1 and args[0].type == T_STR:
                return const_val(len(args[0].const)) if sc.is_const(args[0]) else sc.op1(C["TPLX_OP_SLEN"], T_I64, args[0])
            if name == "str" and len(args) == 1:
                a = args[0]
                if a.type == T_STR:
                    return a
                if a.type == T_I64:
                    return sc.op1(C["TPLX_OP_I2S"], T_STR, a)
                raise UnsupportedUDF("str() of this type")
            if name == "abs" and len(args) == 1 and args[0].type != T_STR:
                a = args[0]
                return sc.op1(C["TPLX_OP_FABS"], T_F64, a) if a.type == T_F64 else sc.op1(C["TPLX_OP_IABS"], T_I64, sc.to_i64(a))
            if name in ("min", "max") and len(args) == 2 and all(a.type != T_STR for a in args):
                x, y = args
                if x.type == T_F64 or y.type == T_F64:
                    x, y = sc.to_f64(x), sc.to_f64(y)
                    c = sc.op2(C["TPLX_OP_FCMP"], T_BOOL, y, x, flags=C["TPLX_CMP_LT" if name == "min" else "TPLX_CMP_GT"])
                else:
                    x, y = sc.to_i64(x), sc.to_i64(y)
                    c = sc.op2(C["TPLX_OP_ICMP"], T_BOOL, y, x, flags=C["TPLX_CMP_LT" if name == "min" else "TPLX_CMP_GT"])
                return sc.select(c, y, x)  # Python: min(x, y) returns y only if y < x
            raise UnsupportedUDF(f"call to {name}()")
        if isinstance(e.func, ast.Attribute):
            obj = self.need(self.expr(e.func.value))
            if isinstance(obj, TupleVal) or obj.type != T_STR:
                raise UnsupportedUDF("method call on non-string")
            m = e.func.attr
            args = [self.need(self.expr(a)) for a in e.args]
            if any(isinstance(a, TupleVal) for a in args):
                raise UnsupportedUDF("tuple argument")

            def want_str(n):
                if len(args) != n or any(a.type != T_STR for a in args):
                    raise UnsupportedUDF(f"str.{m} expects {n} string argument(s)")
            if m == "format":
                if not sc.is_const(obj):
                    raise UnsupportedUDF("format string must be a literal")
                return self.format_braces(obj.const, args)
            if m in ("find", "rfind", "index"):
                want_str(1)
                if m == "index":
                    raise UnsupportedUDF("str.index")
                return sc.op2(C["TPLX_OP_SFIND" if m == "find" else "TPLX_OP_SRFIND"], T_I64, obj, args[0])
            if m in ("lower", "upper"):
                want_str(0)
                if sc.is_const(obj):
                    return const_val(obj.const.lower() if m == "lower" else obj.const.upper())
                return sc.op1(C["TPLX_OP_SLOWER" if m == "lower" else "TPLX_OP_SUPPER"], T_STR, obj)
            if m == "replace":
                want_str(2)
                d = sc.new_vreg(T_STR)
                sc.emit_vals(C["TPLX_OP_SREPLACE"], d, obj, args[0], args[1])
                return Val(T_STR, d)
            if m in ("startswith", "endswith"):
                want_str(1)
                return sc.op2(C["TPLX_OP_SSTARTS" if m == "startswith" else "TPLX_OP_SENDS"], T_BOOL, obj, args[0])
            if m in ("strip", "lstrip", "rstrip"):
                want_str(0)
                fl = {"strip": 3, "lstrip": 1, "rstrip": 2}[m]
                return sc.op1(C["TPLX_OP_SSTRIP"], T_STR, obj, flags=fl)
            raise UnsupportedUDF(f"str.{m}()")
        raise UnsupportedUDF("call expression")
