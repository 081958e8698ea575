/*
 * tplx_ir.h — the stage descriptor ("op program") that replaces the LLVM bitcode a
 * reference TransformStage carries (tuplex/core/include/physical/TransformStage.h:67-514,
 * tuplex/core/src/physical/StageBuilder.cc:1499-1535). A reference stage holds bitcode +
 * symbol names; a non-LLVM backend needs the operator list in a form it can execute, so the
 * planner side (tuplex_b200/frontend.py, or a C++ planner) lowers every UDF of the stage to
 * this flat, typed, predicated register program. The same bytes are consumed by
 *   - the CUDA VM (tuplex_b200/csrc/vm.cuh),
 *   - the CPU oracle (oracle/tplx_oracle.c: tplx_oracle_run_program).
 *
 * Semantics of every op follow the reference codegen/runtime; the file:line each op restates
 * is cited beside it (paths relative to /root/reference/tuplex/).
 *
 * This header is also parsed by tuplex_b200/ir.py (regex over the enum bodies) so that the
 * Python side cannot drift from the C side. Keep one enumerator per line: `NAME = value,`.
 */
#ifndef TPLX_IR_H
#define TPLX_IR_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TPLX_IR_MAGIC 0x58504C54u /* "TPLX" */
#define TPLX_IR_VERSION 8u
#define TPLX_NOSLOT 0xFFFFu
#define TPLX_MAX_COLS 64
#define TPLX_MAX_ACCS 16
#define TPLX_MAX_KEYS 8
/* in_types entry of an "is None" companion input column: TPLX_T_NULLOF | c says "bool column, 1 where Option[T] input column c
 * holds None" (c < TPLX_MAX_COLS). Companions follow the physical columns; the executor fills them from column c's validity
 * bitmap (tplx_column.valid), the caller passes only the physical columns. To the op program a companion is a TPLX_T_BOOL column. */
#define TPLX_T_NULLOF 0x80u
/* flag on a column type where a SCHEMA is given as bytes (tplx_gpu_block_from_partitions col_types): the field is Option[T]
 * and takes part in the row bitmap (Serializer.cc:1041-1059) */
#define TPLX_T_OPTION 0x40u

/* column / value types (python::Type subset on the normal-case path, utils/include/TypeSystem.h) */
enum tplx_type {
    TPLX_T_I64 = 0,
    TPLX_T_F64 = 1,
    TPLX_T_BOOL = 2, /* stored as i64 0/1 in row format (Serializer.cc:1069) and as 8-byte column */
    TPLX_T_STR = 3,  /* column block: uint32 offsets[n+1] + bytes (no NUL); row format: NUL-terminated */
};

/* stage endpoints (TransformStage::outputMode, EndPointMode in core/include/physical/PhysicalStage.h) */
enum tplx_endpoint {
    TPLX_EP_MEMORY = 0,    /* rows out, input order preserved (LocalBackend.cc:1104-1152) */
    TPLX_EP_AGGREGATE = 1, /* AGG_GENERAL: one row out (PipelineBuilder.cc:2525-2608) */
    TPLX_EP_HASH = 2,      /* AGG_BY_KEY / AGG_UNIQUE (PipelineBuilder.cc:1108-1400) */
};

/* accumulator kinds recognised in aggregate UDFs `lambda a, x: a (+) g(x)` (AggregateFunctions.cc:152-243) */
enum tplx_acc_kind {
    TPLX_ACC_SUM_I64 = 0, /* wrapping add (BlockGeneratorVisitor.cc:372-456) */
    TPLX_ACC_SUM_F64 = 1, /* IEEE add, fixed documented tree (DESIGN.md "reduction tree") */
    TPLX_ACC_MIN_I64 = 2,
    TPLX_ACC_MAX_I64 = 3,
    TPLX_ACC_MIN_F64 = 4,
    TPLX_ACC_MAX_F64 = 5,
};

/* compare predicates: signed integer / ordered float (BlockGeneratorVisitor.cc:776-836) */
enum tplx_cmp {
    TPLX_CMP_EQ = 0,
    TPLX_CMP_NE = 1, /* float: FCMP_ONE — false when either side is NaN (reference quirk) */
    TPLX_CMP_LT = 2,
    TPLX_CMP_LE = 3,
    TPLX_CMP_GT = 4,
    TPLX_CMP_GE = 5,
};

/* lazy ASCII case transform carried by a string value (StringFunctions.cc:71-110) */
enum tplx_strflag {
    TPLX_SF_NONE = 0,
    TPLX_SF_LOWER = 1,
    TPLX_SF_UPPER = 2,
};

/* operand-is-constant bits of tplx_instr.flags (upper three bits; the low bits stay op specific).
 * A constant operand is not read from a slot: scalars are the immediate itself, strings are
 * constant-pool views encoded as offset | length << 32.  a <- imm2, b <- imm, c <- imm2. */
enum tplx_constflag {
    TPLX_F_C_CONST = 32,
    TPLX_F_A_CONST = 64,
    TPLX_F_B_CONST = 128,
};

/* slice flags (BlockGeneratorVisitor.cc:4469-4690; stride is always 1 on this path) */
enum tplx_sliceflag {
    TPLX_SL_HAS_START = 1,
    TPLX_SL_HAS_END = 2,
};

/* exception codes used on this path (utils/include/ExceptionCodes.h:24-120) */
enum tplx_exception_code {
    TPLX_EC_SUCCESS = 0,
    TPLX_EC_NORMALCASEVIOLATION = 7,
    TPLX_EC_NULLERROR = 50,
    TPLX_EC_BADPARSE_STRING_INPUT = 70, /* CSV row that does not fit the normal case (ExceptionCodes.h:118) */
    TPLX_EC_PYTHON_PARALLELIZE = 80,
    TPLX_EC_INDEXERROR = 111,
    TPLX_EC_TYPEERROR = 129,
    TPLX_EC_VALUEERROR = 135,
    TPLX_EC_ZERODIVISIONERROR = 136,
};

/*
 * Opcodes (dense numbering: the VM dispatches through a jump table). A value lives in 8-byte slots: scalars (i64 / f64 bits / bool 0-1) take one slot,
 * strings take two consecutive slots: [s] = byte address (generic pointer), [s+1] = len | flags<<32.
 * Every instruction is predicated: it executes for a row iff the row is alive and
 * (guard == TPLX_NOSLOT or slot[guard] != 0). Python if/elif/else and early returns are
 * if-converted by the frontend into guards + TPLX_OP_SEL, so untaken branches can never raise.
 */
enum tplx_op {
    TPLX_OP_NOP = 0,
    /* loads */
    TPLX_OP_LDCOL = 1,  /* dst <- input column imm at this row; flags = tplx_type */
    TPLX_OP_LDI = 2,    /* dst <- imm (i64, f64 bits or bool) */
    TPLX_OP_LDS = 3,    /* dst <- view of constant pool bytes [imm, imm+imm2) */
    TPLX_OP_MOV = 4,    /* dst <- a ; flags = slot count (1|2) */
    TPLX_OP_SEL = 5,    /* dst <- c ? a : b ; flags = slot count (1|2) */
    TPLX_OP_LDROW = 6,  /* dst <- index of this row inside the block (used to merge CPython-resolved rows in order) */
    /* i64 arithmetic: wrapping, no overflow detection (BlockGeneratorVisitor.cc:152-313,372-495) */
    TPLX_OP_IADD = 7,
    TPLX_OP_ISUB = 8,
    TPLX_OP_IMUL = 9,
    TPLX_OP_IFLOORDIV = 10, /* ZeroDivisionError; floor fix-up (LLVMEnvironment.cc:1377-1399) */
    TPLX_OP_IMOD = 11,      /* ZeroDivisionError; floor fix-up (LLVMEnvironment.cc:1402-1430) */
    TPLX_OP_INEG = 12,
    TPLX_OP_IAND = 13,
    TPLX_OP_IOR = 14,
    TPLX_OP_IXOR = 15,
    TPLX_OP_ISHL = 16, /* BlockGeneratorVisitor.cc:612-670 */
    TPLX_OP_ISHR = 17,
    TPLX_OP_IABS = 18,
    /* f64 arithmetic: single IEEE-754 ops, no contraction (BlockGeneratorVisitor.cc:152-584) */
    TPLX_OP_FADD = 19,
    TPLX_OP_FSUB = 20,
    TPLX_OP_FMUL = 21,
    TPLX_OP_FDIV = 22,      /* ZeroDivisionError when divisor == 0.0 (divisionInst :497-530) */
    TPLX_OP_FMOD = 23,      /* frem + sign fix (LLVMEnvironment.cc:1415-1422); ZeroDivisionError */
    TPLX_OP_FNEG = 24,
    TPLX_OP_FFLOORDIV = 25, /* both sides fptosi, floor-div, sitofp (integerDivisionInst :360-365) */
    TPLX_OP_FABS = 26,
    /* conversions (FunctionRegistry.cc:83-148, upCast) */
    TPLX_OP_I2F = 27, /* sitofp */
    TPLX_OP_F2I = 28, /* fptosi (trunc) — int(f64) */
    /* comparisons -> bool; flags = tplx_cmp */
    TPLX_OP_ICMP = 29,
    TPLX_OP_FCMP = 30,
    /* logical on 0/1 values */
    TPLX_OP_BAND = 31,
    TPLX_OP_BOR = 32,
    TPLX_OP_BNOT = 33,
    /* strings (ASCII bytes; FunctionRegistry.cc / runtime/src/Runtime.cc / StringFunctions.cc) */
    TPLX_OP_SLEN = 34,     /* len(s) */
    TPLX_OP_SFIND = 35,    /* s.find(b): strstr (FunctionRegistry.cc:2165-2188); -1 if absent */
    TPLX_OP_SRFIND = 36,   /* s.rfind(b): std::string::rfind (Runtime.cc:387-397) */
    TPLX_OP_SIN = 37,      /* a in b -> strstr(b, a) != NULL (BlockGeneratorVisitor.cc:838-880) */
    TPLX_OP_SEQ = 38,      /* strcmp == 0 ; flags bit0 = negate (!=) */
    TPLX_OP_SSLICE = 39,   /* a[b:c], flags = tplx_sliceflag (processSliceIndex :4618-4690) */
    TPLX_OP_SINDEX = 40,   /* a[b] one-char string; IndexError (BlockGeneratorVisitor.cc:3869-3903) */
    TPLX_OP_SLOWER = 41,   /* lazy flag (StringFunctions.cc:71-89) */
    TPLX_OP_SUPPER = 42,   /* lazy flag (StringFunctions.cc:91-108) */
    TPLX_OP_SREPLACE = 43, /* a.replace(b, c), materialises (Runtime.cc:401-540) */
    TPLX_OP_SCONCAT = 44,  /* a + b, materialises (BlockGeneratorVisitor.cc:381-436) */
    TPLX_OP_SFMTD = 45,    /* '%[0][w]d' % a : snprintf %d of (int)a, imm=width, flags bit0=zero pad,
                              constant prefix/suffix via b/c string slots (BlockGeneratorVisitor.cc:675-775) */
    TPLX_OP_S2I = 46,      /* int(s): fast_atoi64 (Runtime.cc:319-341, StringUtils.cc:22-63); ValueError */
    TPLX_OP_STRUTH = 47,   /* bool(s): len > 0 */
    TPLX_OP_SSTARTS = 48,  /* a.startswith(b) */
    TPLX_OP_SENDS = 49,    /* a.endswith(b) */
    TPLX_OP_I2S = 50,      /* str(i64), materialises */
    TPLX_OP_SSTRIP = 51,   /* a.strip() whitespace view; flags bit0 = left, bit1 = right */
    /* row control */
    TPLX_OP_FILTER = 52, /* alive &= slot[a] != 0 (PipelineBuilder.cc:615-700) */
    TPLX_OP_RAISE = 53,  /* unconditional (guarded) exception imm = code */
    TPLX_OP_S2F = 54,    /* float(s): fast_atod behind the runtime's trim (Runtime.cc:343-365, StringUtils.cc:71-163); ValueError */
    /* fused forms of two idioms the planner recognises (what inlining + select folding give the reference's LLVM -O2,
     * LLVMOptimizer.cc:119-191); each is defined as the primitive sequence it replaces */
    TPLX_OP_SFINDE = 55,  /* i = a.find(b); dst <- i < 0 ? len(a) : i          ("split at marker, else whole string") */
    TPLX_OP_SRFINDK = 56, /* i = a.rfind(b); dst <- i < 0 ? 0 : i + imm2       ("start after the last separator"); a is never constant */
};

/* 32-byte instruction */
typedef struct tplx_instr {
    uint8_t op;     /* tplx_op */
    uint8_t flags;  /* op specific */
    uint16_t dst;   /* destination slot or TPLX_NOSLOT */
    uint16_t a;     /* source slots */
    uint16_t b;
    uint16_t c;
    uint16_t guard; /* bool slot or TPLX_NOSLOT */
    uint16_t opidx; /* index into the stage's operator-id table (exception attribution) */
    uint16_t pad;
    int64_t imm;
    int64_t imm2;
} tplx_instr;

typedef struct tplx_outcol {
    uint16_t slot;   /* value slot at program end */
    uint8_t type;    /* tplx_type */
    uint8_t null_of; /* 0, or 1 + k: this (hidden, TPLX_T_BOOL) column is 1 where output column k — an Option[T] column — holds None;
                        the executor turns it into column k's validity bitmap (tplx_gpu_result_fetch_validity).
                        HASH endpoint: allowed on hidden bool columns behind the keys only, and k must be one of the first n_keys
                        columns (at most one companion per key). Rows whose flag is 1 form key k's None group: the key's value
                        slot is then ignored, None differs from every value (0, "", False), and the hash result carries
                        the key column with a validity bitmap (placeholder 0 / "" under None). */
} tplx_outcol;

typedef struct tplx_acc {
    uint8_t kind;  /* tplx_acc_kind */
    uint8_t pad;
    uint16_t slot; /* per-row value g(x) */
    uint32_t pad2;
    int64_t init;  /* initial value bits (i64 or f64) — applied once per block, like the per-task
                      intermediate in BlockBasedTaskBuilder.cc:185-206 */
} tplx_acc;

/*
 * Serialized stage descriptor layout (little endian, 8-byte aligned sections):
 *   tplx_stage_header
 *   uint8_t  in_types[n_in_cols]      (padded to 8)
 *   tplx_outcol out_cols[n_out_cols]  (padded to 8)   -- MEMORY: output row; HASH: key columns first
 *   tplx_acc accs[n_accs]
 *   int64_t  opids[n_ops]             -- reference operator ids (LogicalOperator.h:52-59, start 100000)
 *   tplx_instr instrs[n_instr]
 *   uint8_t  const_pool[const_bytes]  (padded to 8)
 *   uint8_t  prefilter[prefilter_bytes]  -- optional nested stage descriptor (same layout), see below
 *   uint8_t  fused[fused_bytes]          -- optional tplx_fused_header + predicates + terms, see below
 *
 * Prefilter (selective pipelines): a MEMORY stage whose single output column is the row index
 * (TPLX_OP_LDROW) of the rows that survive the leading, selective part of the pipeline. The executor runs
 * it first and then runs THIS stage densely over the surviving row list only (late materialisation: the
 * columns that only survivors need are never read for the other rows). It is an execution hint: running
 * this stage over all rows gives the same result, which is what the oracle does.
 */
/*
 * Fused scan-aggregate hint (AGGREGATE endpoint): when every operator of the stage is a filter made of range
 * comparisons between one fixed-width column and constants, and every accumulator is a sum of a constant, a column
 * or a product of two columns (the TPC-H Q6 class, benchmarks/tpch/Q06/runtuplex.py:96-99), the planner ALSO
 * states the stage in this closed form. The executor may then run a dedicated streaming kernel instead of the VM.
 * Like the prefilter it is an execution hint: same rows, same per-row IEEE operations, same reduction tree — the
 * oracle ignores it and the parity tests compare the two.
 */
#define TPLX_FUSED_MAGIC 0x31415346u /* "FSA1" */
enum tplx_fused_predflag {
    TPLX_FP_F64 = 1,      /* compare as f64 (ordered), else signed i64 */
    TPLX_FP_HAS_LO = 2,
    TPLX_FP_LO_INCL = 4,
    TPLX_FP_HAS_HI = 8,
    TPLX_FP_HI_INCL = 16,
    TPLX_FP_CAST = 32,    /* column is i64, converted with sitofp before an f64 compare */
};
enum tplx_fused_termop {
    TPLX_FT_CONST = 0,    /* g(x) = imm */
    TPLX_FT_COL = 1,      /* g(x) = col_a */
    TPLX_FT_MUL = 2,      /* g(x) = col_a * col_b (single IEEE multiply, or wrapping i64 multiply) */
};
typedef struct tplx_fused_pred {
    uint32_t col;
    uint32_t flags; /* tplx_fused_predflag */
    int64_t lo, hi; /* i64 values or f64 bits */
} tplx_fused_pred;
typedef struct tplx_fused_term {
    uint32_t kind;   /* tplx_acc_kind, same order as the stage's accumulators */
    uint32_t op;     /* tplx_fused_termop */
    uint32_t col_a, col_b;
    uint32_t cast_a, cast_b; /* 1: i64 column converted with sitofp first */
    int64_t imm;
} tplx_fused_term;
typedef struct tplx_fused_header {
    uint32_t magic;
    uint32_t n_preds;
    uint32_t n_terms;
    uint32_t pad;
} tplx_fused_header;
#define TPLX_MAX_FUSED_PREDS 8

/*
 * String-scan hint (MEMORY endpoint; used for the prefilter stage of a selective pipeline): when the whole stage is a chain of
 * filters, each of one of the closed forms below, the planner ALSO states it as a list of terms (carried in the `fused` section
 * of that stage with TPLX_SCAN_MAGIC). The executor may then evaluate the terms with a dedicated kernel instead of interpreting
 * the program. An execution hint like the two above: same rows kept, same exception rows (code, operator), evaluated in program
 * order so that a row raises only in terms it reaches; the oracle ignores it and the parity tests compare both paths.
 *   CONTAINS    needle in column (column optionally lower()/upper()-ed), optionally negated          SLOWER/SUPPER + SIN (+ BNOT) + FILTER
 *   FIELD_INT   i = s.find(marker); head = s[: i if i >= 0 else len(s)]; j = head.rfind(sep);
 *               v = int(head[(0 if j < 0 else j + skip):]);  v <cmp> imm                             SFINDE SSLICE SRFINDK SSLICE S2I ICMP FILTER
 *               (ValueError of int() -> exception row attributed to operator opidx_val)
 *   FIXED       fixed-width column <cmp> imm (signed i64 / ordered f64)                              ICMP|FCMP + FILTER
 */
#define TPLX_SCAN_MAGIC 0x31435353u /* "SSC1" */
#define TPLX_MAX_SCAN_TERMS 8
enum tplx_scan_kind {
    TPLX_SK_CONTAINS = 0,
    TPLX_SK_FIELD_INT = 1,
    TPLX_SK_FIXED = 2,
};
enum tplx_scan_flag {
    TPLX_SCF_CASE_MASK = 3, /* tplx_strflag applied to the column value */
    TPLX_SCF_NEGATE = 4,    /* CONTAINS: keep the row when the needle is absent */
    TPLX_SCF_F64 = 8,       /* FIXED: compare as f64 (ordered), else signed i64 */
};
typedef struct tplx_scan_term {
    uint32_t kind;      /* tplx_scan_kind */
    uint32_t col;       /* input column */
    uint32_t flags;     /* tplx_scan_flag */
    uint32_t cmp;       /* tplx_cmp of (value <cmp> imm): FIELD_INT, FIXED */
    int64_t imm;        /* i64 or f64 bits */
    uint64_t needle;    /* constant-pool view (offset | length << 32): CONTAINS needle / FIELD_INT marker */
    uint64_t sep;       /* FIELD_INT: separator (constant-pool view) */
    int64_t skip;       /* FIELD_INT: added to the separator position */
    uint32_t opidx_val; /* operator index of the part that can raise (int()) */
    uint32_t opidx_filter;
    uint64_t pad;
} tplx_scan_term;
typedef struct tplx_scan_header {
    uint32_t magic;
    uint32_t n_terms;
    uint64_t pad;
} tplx_scan_header;

typedef struct tplx_stage_header {
    uint32_t magic;
    uint32_t version;
    uint32_t total_bytes;
    uint16_t n_in_cols;
    uint16_t n_out_cols;
    uint16_t n_accs;
    uint16_t n_keys;      /* HASH endpoint: first n_keys out_cols are the key; hidden `is None` companions of Option keys
                             (tplx_outcol.null_of) may follow them */
    uint16_t n_ops;
    uint16_t n_slots;     /* register file size in 8-byte slots */
    uint32_t n_instr;
    uint32_t const_bytes;
    uint8_t endpoint;     /* tplx_endpoint */
    uint8_t pad0;
    uint16_t hidden_out_cols; /* trailing output columns that are executor-internal (row index of each output
                                 row, used to number exception rows when a prefilter ran); never handed out */
    uint32_t scratch_bytes;   /* per-row scratch for materialised strings */
    uint32_t prefilter_bytes; /* size of the nested prefilter stage descriptor, 0 = none */
    uint32_t fused_bytes;     /* size of the optional closed-form hint: tplx_fused_header ... (AGGREGATE) or tplx_scan_header ... (MEMORY); 0 = none */
} tplx_stage_header;

#ifdef __cplusplus
}
#endif
#endif /* TPLX_IR_H */
