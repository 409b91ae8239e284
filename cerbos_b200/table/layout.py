"""Binary layout shared by the host flattener, the batch encoder, the CUDA kernels and
the C oracle: section ids of the table blob, value tags, bytecode opcodes.

This module is the single source of truth; ``python -m cerbos_b200.table.layout``
regenerates ``include/cerbos_b200_format.h`` (tests check the header is in sync).

Table blob (little endian, every section 16-byte aligned):
    BlobHeader { u32 magic; u32 version; u32 n_sections; u32 flags; u64 total_bytes; u64 reserved }
    SectionDesc[n_sections] { u32 id; u32 elem_bytes; u64 offset; u64 n_bytes }
    sections...
"""
from __future__ import annotations

MAGIC = 0x32425243  # 'CRB2'
VERSION = 17
ALIGN = 16

NONE32 = 0xFFFFFFFF
NONE16 = 0xFFFF
ROLE_ANY = 0xFFFF          # row.role: matches any role ("*")
ROLE_UNKNOWN = 0xFFFFFFFE  # request role not in the table's role dictionary
ROLE_PAD = 0xFFFFFFFF      # unused role column entry
SCOPE_NONE = 0x7FFFFFFF    # request scope that resolves to nothing
SCOPE_INEXACT_BIT = 0x80000000  # lenient: hdr scope is the nearest known ancestor, not the request's own scope
KIND_CLASS_CSR_BIT = 0x80000000  # hdr0.kind_class: bit clear = the single matching resource pattern id (KIND_NONE =
KIND_NONE = 0x7FFFFFFF           # matches nothing); bit set = index into the class_off / class_pats CSR

# ---- sections -----------------------------------------------------------------------------------------
SECTIONS = {
    "META": 1,            # u32[META_WORDS]
    "SCOPE_PARENT": 2,    # u32[n_scopes]   nearest ancestor scope present in the dictionary, or NONE32
    "SCOPE_FLAGS": 3,     # u32[n_scopes]   bit0 in principalScopeMap, bit1 in resourceScopeMap, bits 4-5 scope permissions
    "RES_BLOCK_MAP": 4,   # u32[n_versions*n_respats*n_scopes] -> block id | NONE32
    "RES_EXISTS": 5,      # u8 [n_versions*n_respats*n_scopes] bit0 RESOURCE-kind row exists, bit1 any row exists
    "PRIN_BLOCK_MAP": 6,  # u32[n_versions*n_principals*n_scopes] -> block id | NONE32
    "PRIN_EXISTS": 7,     # u8 [n_versions*n_scopes]  any PRINCIPAL-kind row with (version, scope)
    "PRIN_OF_STRING": 8,  # u32[n_strings] string id -> principal index | NONE32
    "BLOCKS": 9,          # Block[n_blocks] {u32 row_start, n_rows, cond_base, n_conds}
    "ROWS": 10,           # Row[n_rows] 16 B; rows of a block that differ only in their action pattern are merged
    "CONDS": 11,          # {u32 code_off, code_len, flat_off, flat_info}[n_conds]  (offsets in instructions)
    "CODE": 12,           # Instr[n_code] 8 B {u8 op; u8 a; u16 b; u32 c}
    "CONSTS": 13,         # Const[n_consts] 16 B {u32 tag; u32 pad; u64 bits}
    "THEAP": 14,          # u64[] constant lists / maps (NaN-boxed V64 elements)
    "STR_OFF": 15,        # u32[n_strings+1]
    "STR_BYTES": 16,      # u8[]
    "ROLE_PARENTS_OFF": 17,  # u32[n_scopes*n_roles+1] CSR offsets (only when has_parent_roles)
    "ROLE_PARENTS": 18,   # u32[] role ids (transitive closure, per (scope, role))
    "ROLEPOL_OFF": 19,    # u32[n_versions*n_scopes+1] CSR into ROLEPOL_ENTRIES
    "ROLEPOL_ENTRIES": 20,  # {u32 role; u32 rule_start; u32 n_rules; u32 pad}
    "ROLEPOL_RULES": 21,  # {u32 respat; u32 cond (global id+1, 0 none); u32 apat_start; u32 n_apats}
    "ROLEPOL_APATS": 22,  # u32[] action pattern ids
    "ROW_APATS": 24,      # u32[] action pattern ids of the (merged) rows (CSR via row.pat_start / n_pats)
    "BLOCK_SLOTS_OFF": 25,  # u32[n_blocks+1] CSR: attribute slots read by the conditions of a block (prefetch list)
    "BLOCK_SLOTS": 26,    # u32[]
    "CONSTS_V64": 23,     # u64[n_consts] NaN-boxed form of each constant for the flat fast path (FLAT_NOT_FAST if none)
    # derived roles of every resource policy block (effectiveDerivedRoles bookkeeping, ruletable.go:936-979)
    "DR_OFF": 27,         # u32[n_blocks+1] CSR into DR_ENTRIES
    "DR_ENTRIES": 28,     # {u32 name index (MANIFEST derived_roles, sorted); cond (global id + 1, 0 none); parents start; n parents}
    "DR_PARENTS": 29,     # u32[] parent role ids (ROLE_ANY for "*")
    "DR_NAME_STR": 30,    # u32[n derived role names] string id of each name (runtime.effectiveDerivedRoles in conditions)
    # rule outputs (present only when the table declares outputs; blocks holding an output row keep one row per rule action)
    "ROW_OUT": 31,        # u32[n_rows] OUT_ENTRIES index of the row | NONE32
    "OUT_ENTRIES": 32,    # {u32 src id (MANIFEST output_sources); activated code_off | NONE32; not-met code_off | NONE32; flags OUT_UNLOWERED_*}
    "MANIFEST": 100,      # JSON (host only): dictionaries + slot paths for the batch encoder
}

META_WORDS = 32
META = {name: i for i, name in enumerate([
    "n_versions", "n_respats", "n_scopes", "n_principals", "n_roles", "n_apats", "n_blocks", "n_rows",
    "n_conds", "n_code", "n_consts", "n_slots", "n_strings", "has_role_policies", "has_parent_roles",
    "has_principal_policies", "max_stack", "max_loop_depth", "n_vars", "theap_words", "uses_pid", "uses_now",
    "max_scope_depth", "direct_kinds", "block_shapes", "uses_runtime", "n_dr_names", "n_output_rows", "n_unlowered_outputs",
])}
IMAGE_SECTIONS = 33   # section ids below this travel in the device image (TableLayout::off); MANIFEST is host-only

SCOPE_FLAG_PRINCIPAL = 1
SCOPE_FLAG_RESOURCE = 2
SCOPE_PERM_SHIFT = 4

EXISTS_RESOURCE_KIND = 1
EXISTS_ANY_ROW = 2

ROW_FLAG_PRINCIPAL = 1

EFFECT_ALLOW = 1
EFFECT_DENY = 2

# ---- 8-byte NaN-boxed values (attribute columns, heap elements) ------------------------------------------
# doubles are stored raw; everything else is boxed: bits 63..48 = 0xFFF0 | tag, payload = low 48 bits.
V64_BOX_BASE = 0xFFF0
V64_NULL = 1
V64_BOOL = 2
V64_STRING = 3    # payload = string id
V64_LIST = 4      # payload = heap word offset (bit 47 set = batch heap, clear = table heap)
V64_MAP = 5
V64_ABSENT = 6    # slot only: the last path segment is missing from its (map) parent
V64_ERROR = 7     # slot only: path traverses a missing / non-map value
V64_INT = 8       # payload = 48-bit two's complement (constants in the table heap only)
V64_HEAP_BATCH_BIT = 1 << 47
V64_CANON_NAN = 0x7FF8000000000000

# ---- interpreter value tags ---------------------------------------------------------------------------------
TAGS = {name: i for i, name in enumerate([
    "ERR", "NULL", "BOOL", "INT", "UINT", "DOUBLE", "STRING", "LIST", "MAP", "TS", "DUR", "BYTES", "TYPE",
    "SPIFFE_ID", "SPIFFE_TD",     # conditions/types/spiffe.go: a validated SPIFFE id string; a trust domain name (payload: a string reference)
])}

# ---- bytecode ---------------------------------------------------------------------------------------------------
OPS = {name: i for i, name in enumerate([
    "RET",          # result = TOS
    "CONST",        # push consts[c]
    "SLOT",         # push slot[c]            (ABSENT / ERROR -> ERR)
    "HAS_SLOT",     # push BOOL(slot[c] present) ; ERROR slot -> ERR
    "PID",          # push STRING(hdr.principal_id)
    "NOW",          # push TS(batch now)
    "VAR",          # push loop variable a
    "SELECT",       # TOS map . key(string id c)
    "HAS",          # TOS map has key c -> BOOL
    "INDEX",        # [container, key] -> value
    "EQ", "NE", "LT", "LE", "GT", "GE",
    "ADD", "SUB", "MUL", "DIV", "MOD", "NEG", "NOT",
    "IN",           # [x, container] -> BOOL
    "SIZE",
    "STARTS_WITH", "ENDS_WITH", "CONTAINS",   # [s, t] -> BOOL
    "JF_KEEP",      # if TOS is BOOL false: pc = c (TOS kept)
    "JT_KEEP",      # if TOS is BOOL true:  pc = c (TOS kept)
    "AND", "OR",    # [a, b] -> 3-valued combine with cel-go error absorption
    "JMP",          # pc = c
    "TERN",         # pop cond: true -> fallthrough ; false -> pc = c ; else push ERR, pc = b (end)
    "HAS_INTERSECTION", "IS_SUBSET",   # [a, b] lists -> BOOL
    "LOOP_INIT",    # pop range; a = var slot, b = kind (LOOP_*), c = end pc
    "LOOP_NEXT",    # pop body result; a = var slot, b = kind, c = body pc
    "TO_COND",      # TOS -> BOOL(TOS is BOOL true)   (error / non-bool -> false; ruletable.go:1425-1441)
    "COND_NOT",     # TOS BOOL -> !TOS
    "NOERR",        # TOS -> BOOL(TOS is not ERR)     (has(V.x) on an inlined variable)
    "INT", "UINT", "DOUBLE", "TIMESTAMP", "DURATION", "DYN",  # conversions of TOS
    "TYPE_EQ",      # unused placeholder (reserved)
    # super-instructions (fused forms of the sequences above; same results)
    "CMP_SLOT_CONST",   # push cmp(a=EQ..GE as op index)(slot[b], consts[c])
    "CMP_SLOT_SLOT",    # push cmp(a)(slot[b], slot[c])
    "CMP_SLOT_PID",     # push cmp(a)(slot[b], P.id)
    "IN_SLOT_CONST",    # push slot[b] in consts[c]
    "IN_CONST_SLOT",    # push consts[c] in slot[b]
    "IN_IP_RANGE",      # TOS string ip -> BOOL(ip in CIDR at theap[c..c+3] = {family 4|6, prefix bits, hi64, lo64})
    # hierarchy(s[, delim]) values never materialise: the functions over them are fused (conditions/types/hierarchy.go)
    "HIER_REL",         # [s, t] strings -> BOOL: a = HIER_* relation of hierarchy(s, delim b) with hierarchy(t, delim c)
    "HIER_SIZE",        # [s] -> INT segments of hierarchy(s, delim b)
    "HIER_CA",          # a = 0: [s, t] -> INT size of s.commonAncestors(t); a = 1: [s, t, z] -> BOOL(commonAncestors == hierarchy(z));
                        #        delimiters b (s), c & 0xFFFF (t), c >> 16 (z)
    "IN_SPLIT",         # [x, s] -> BOOL(x in s.split(delim b)): the token list never materialises (ext strings split)
    "TS_GET",           # TOS timestamp / duration -> INT: a = TS_FIELDS getter (0xFF: always an error), c = fixed offset east of UTC
                        # in seconds (int32), b = 1 when a zone argument was given (then a duration operand is an error);
                        # b = 2: an IANA zone -- c = theap offset of its transition table [n, first, last, (utc second, offset)...]
    # values made at run time (per-thread scratch arena on the device)
    "FN",               # a = FN id, b = argument count n: [arg0 .. argn-1] -> result (string / list functions below)
    "MKLIST",           # c = n: [e0 .. en-1] -> list
    "MKMAP",            # c = n: [k0, v0 .. kn-1, vn-1] -> map
    "LOOP_PRED",        # TOS = predicate of a filtering map / transformList / transformMap / transformMapEntry: true -> pop and
                        # fall through to the transform; false -> skip this iteration; else error. c = pc of the LOOP_NEXT
    "MATCHES",          # TOS string -> BOOL: RE2 search with the byte-level DFA at theap[c] (cel/regex_dfa.py)
    "RUNTIME_EDR",      # push runtime.effectiveDerivedRoles: the derived roles in force for the policy being evaluated (list of strings)
])}
# FN FORMAT: fmt.format(args) with a constant fmt (ext.Strings).  Its first argument is an INT constant: the THEAP offset of the
# parsed clause record | mode << 32.  FORMAT_ARGS_STACK: the remaining arguments are the list literal's elements;
# FORMAT_ARGS_LIST: the one remaining argument is the list.  The clause record is [n items, then one word per item]; an item is
# a literal run (verb byte 0, table string id in bits 32..63) or a clause (verb byte 's' 'd' 'f' 'e' 'b' 'x' 'X' 'o', precision
# in bits 16..31, FMT_PREC_DEFAULT = none given)
FORMAT_ARGS_STACK = 0
FORMAT_ARGS_LIST = 1
FMT_PREC_DEFAULT = 0xFFFF
# FN ids: string functions first (cel-go ext.Strings), list functions from EXCEPT on (ext.Lists, Cerbos except / intersect)
FNS = {name: i for i, name in enumerate([
    "LOWER", "UPPER", "TRIM", "STR_REVERSE", "CHARAT", "INDEXOF", "LASTINDEXOF", "SUBSTRING", "REPLACE", "SPLIT", "JOIN",
    "HIER_JOIN",        # hierarchy(list of strings): the parts joined by U+001F (the delimiter the fused hierarchy ops then use)
    "HIER_AT",          # [s, i, delim]: hierarchy(s, delim)[i]
    "TO_BYTES",         # bytes(string | bytes)
    "B64ENC", "B64DEC", # base64.encode(bytes) -> string, base64.decode(string) -> bytes (std alphabet, padding optional)
    "EXCEPT", "INTERSECT", "SORT", "REVERSE", "SLICE", "FLATTEN", "DISTINCT", "RANGE",
    # SPIFFE (conditions/types/spiffe.go); a matcher never exists as a value: matcher(arg).matchesID(x) is one fused function
    "SPIFFE_ID", "SPIFFE_TD", "SPIFFE_PATH", "SPIFFE_TD_OF", "SPIFFE_MEMBER", "SPIFFE_TD_ID", "SPIFFE_TD_NAME", "SPIFFE_IDSTR",
    "SPIFFE_MATCH_ANY", "SPIFFE_MATCH_EXACT", "SPIFFE_MATCH_ONEOF", "SPIFFE_MATCH_TD",
    # cel-go ext.Math (conditions/cel.go:62-75 enables it): scalars in, a scalar out
    "MATH_GREATEST", "MATH_LEAST", "MATH_CEIL", "MATH_FLOOR", "MATH_ROUND", "MATH_TRUNC", "MATH_ABS", "MATH_SIGN", "MATH_ISNAN", "MATH_ISINF",
    "MATH_ISFINITE", "MATH_BITAND", "MATH_BITOR", "MATH_BITXOR", "MATH_BITNOT", "MATH_SHL", "MATH_SHR", "MATH_SQRT",
    "TO_STRING",        # string(x): strings, ints, uints, bools, valid UTF-8 bytes, integral doubles below 2^53 (the rest is flagged)
    "TYPE_OF",          # type(x) -> a TYPE value (payload: TYPE_CODES); type names are TYPE constants, compared by payload
    "TO_BOOL",          # bool(x): a bool, or a string strconv.ParseBool reads ("1" "t" "T" "TRUE" "true" "True" / "0" "f" "F" "FALSE" "false" "False")
    "QUOTE",            # strings.quote(s): s in double quotes, \a \b \f \n \r \t \v \\ and \" escaped
    "FORMAT",           # [record, args...]: fmt.format(args) by a parsed clause record (FORMAT_ARGS_* below)
])}
# payload of a TYPE value (type(x), the identifiers int / string / ... in an expression)
TYPE_CODES = {"bool": 1, "int": 2, "uint": 3, "double": 4, "string": 5, "bytes": 6, "list": 7, "map": 8, "null_type": 9,
              "google.protobuf.Timestamp": 10, "google.protobuf.Duration": 11, "type": 12}
TS_FIELDS = {name: i for i, name in enumerate(["getFullYear", "getMonth", "getDayOfYear", "getDayOfMonth", "getDate", "getDayOfWeek",
                                               "getHours", "getMinutes", "getSeconds", "getMilliseconds"])}
HIER_RELS = {name: i for i, name in enumerate(["ancestorOf", "descendentOf", "immediateChildOf", "immediateParentOf", "siblingOf", "overlaps", "equals"])}

# Flat fast-path conditions: a condition in disjunctive normal form over "terms".  A term is 16 bytes (two CODE
# slots): {u8 op; u8 flags; u8 xk; u8 yk; u32 x; u32 y; u16 xa; u16 ya}.  Its value is tri-state (true / false /
# error); the literal it contributes is selected by flags: T ("is BOOL true"), F ("is BOOL false").  Terms are
# AND-ed into groups (FLAT_GROUP_END closes a group), groups are OR-ed; CONDS.flat_info = n_terms | FLAT_DNF << 16
# | negate << 24 (final negation: a top-level `none`); 0 = the condition has no flat form.
FLAT_DNF = 3
TERM_OPS = {name: i for i, name in enumerate([
    "CMP", "IN", "STARTS", "ENDS", "CONTAINS", "HAS", "INTERSECTS", "SUBSET",
    # operand-specialised forms of CMP / IN chosen by bytecode.compile_flat (S = attribute slot, C = scalar constant or
    # constant list of scalars, P = principal id): same semantics, straight-line device code per shape
    "EQ_SS", "EQ_SC", "EQ_SP", "ORD_SS", "ORD_SC", "IN_SC", "IN_CS", "IN_SS",
])}
TERM_CI_MASK = 0x07        # flags: compare index for CMP (0 EQ, 2 LT, 3 LE, 4 GT, 5 GE)
TERM_LIT_F = 0x20          # flags: literal is "term is BOOL false" (else "is BOOL true")
TERM_GROUP_END = 0x40      # flags: last term of its AND-group
OPK = {name: i for i, name in enumerate(["SLOT", "CONST", "PID", "SLOT_ELEM", "SLOT_SIZE"])}
FLAT_NOT_FAST = ((V64_BOX_BASE | 15) << 48)   # CONSTS_V64 entry: constant has no 8-byte fast form
FLAT_MAX_TERMS = 24

LOOP_ALL = 0
LOOP_EXISTS = 1
LOOP_EXISTS_ONE = 2
LOOP_MAP = 3          # collecting comprehensions: kinds >= LOOP_MAP build a list / map in the scratch arena
LOOP_FILTER = 4
LOOP_TMAP = 5         # transformMap: {key of the iteration: transform}
LOOP_TENTRY = 6       # transformMapEntry: the transform yields a map whose entries are merged
LOOP_SORTBY = 7       # sortBy: the elements ordered by the key the body yields (stable)

CMP_INDEX = {"_==_": 0, "_!=_": 1, "_<_": 2, "_<=_": 3, "_>_": 4, "_>=_": 5}

MAX_STACK = 16
MAX_LOOP_DEPTH = 2
MAX_VARS = 4
MAX_CHAIN = 8       # scope chain length supported on device (depth+1)
MAX_ROLE_COLS = 16
MAX_CLASS_PATS = 8  # resource patterns one request kind may match

# decision metadata: where ActionEffect.Policy comes from (ruletable.go:913-922, 1082-1095)
META_SRC = {"NO_MATCH": 0, "PRINCIPAL_POLICY": 1, "RESOURCE_POLICY": 2, "NO_MATCH_FOR_SCOPE_PERMISSIONS": 3, "ROLE_POLICY": 4}

# rule outputs (cgpu_check_outputs).  OUT_ENTRIES.flags: the activated / not-met expression has no device program; a
# request that visits it fails the call with CGPU_ERR_UNSUPPORTED.
OUT_UNLOWERED_ACTIVATED = 1
OUT_UNLOWERED_NOT_MET = 2
# Output records: every request owns `stride` bytes {u32 bytes_needed; u32 n_entries} + entries in emission order.  An entry
# is {u16 action index; u16 pad; u32 src id} + one value; a value is a tag byte + payload (little endian, unaligned):
#   BOOL u8 | INT i64 | UINT u64 | DOUBLE f64 | STRING / BYTES u32 length + bytes | TIMESTAMP / DURATION i64 nanoseconds |
#   LIST u32 n + n values | MAP u32 n + n (key, value) pairs | NO_VALUE (evaluation error), NULL, NOT_CONVERTIBLE: nothing.
# Values are CEL-typed; the conversion to google.protobuf.Value happens on the host (cerbos_b200/outputs.py).
OUT_TAGS = {name: i for i, name in enumerate([
    "NO_VALUE", "NULL", "BOOL", "INT", "UINT", "DOUBLE", "STRING", "BYTES", "TIMESTAMP", "DURATION", "LIST", "MAP",
    "NOT_CONVERTIBLE",
])}
OUT_RECORD_HEADER = 8
OUT_ENTRY_HEADER = 8
OUT_MAX_STACK = 32  # evaluation stack of a value program (literal maps and lists of a rule output sit on it whole)
OUT_MAX_DEPTH = 8   # nesting of lists / maps an output value may have on the device (deeper: CGPU_ERR_UNSUPPORTED)

# batch flags (cgpu_batch.flags)
BATCH_FLAG_LENIENT = 1


def c_header() -> str:
    out = ["/* GENERATED by `python -m cerbos_b200.table.layout` -- do not edit. */",
           "#ifndef CERBOS_B200_FORMAT_H", "#define CERBOS_B200_FORMAT_H", "#include <stdint.h>", ""]

    def d(name, val, hexa=False):
        if hexa:
            out.append(f"#define {name} 0x{val:X}u" if val <= 0xFFFFFFFF else f"#define {name} 0x{val:X}ull")
        else:
            out.append(f"#define {name} {val}")

    d("CB_MAGIC", MAGIC, True)
    d("CB_VERSION", VERSION)
    d("CB_NONE32", NONE32, True)
    d("CB_NONE16", NONE16, True)
    d("CB_ROLE_ANY", ROLE_ANY, True)
    d("CB_ROLE_UNKNOWN", ROLE_UNKNOWN, True)
    d("CB_ROLE_PAD", ROLE_PAD, True)
    d("CB_SCOPE_NONE", SCOPE_NONE, True)
    d("CB_SCOPE_INEXACT_BIT", SCOPE_INEXACT_BIT, True)
    d("CB_KIND_CLASS_CSR_BIT", KIND_CLASS_CSR_BIT, True)
    d("CB_KIND_NONE", KIND_NONE, True)
    out.append("")
    for k, v in SECTIONS.items():
        d(f"CB_SEC_{k}", v)
    out.append("")
    d("CB_META_WORDS", META_WORDS)
    for k, v in META.items():
        d(f"CB_META_{k.upper()}", v)
    out.append("")
    d("CB_SCOPE_FLAG_PRINCIPAL", SCOPE_FLAG_PRINCIPAL)
    d("CB_SCOPE_FLAG_RESOURCE", SCOPE_FLAG_RESOURCE)
    d("CB_SCOPE_PERM_SHIFT", SCOPE_PERM_SHIFT)
    d("CB_EXISTS_RESOURCE_KIND", EXISTS_RESOURCE_KIND)
    d("CB_EXISTS_ANY_ROW", EXISTS_ANY_ROW)
    d("CB_ROW_FLAG_PRINCIPAL", ROW_FLAG_PRINCIPAL)
    d("CB_EFFECT_ALLOW", EFFECT_ALLOW)
    d("CB_EFFECT_DENY", EFFECT_DENY)
    out.append("")
    d("CB_V64_BOX_BASE", V64_BOX_BASE, True)
    for k in ("NULL", "BOOL", "STRING", "LIST", "MAP", "ABSENT", "ERROR", "INT"):
        d(f"CB_V64_{k}", globals()[f"V64_{k}"])
    d("CB_V64_HEAP_BATCH_BIT", V64_HEAP_BATCH_BIT, True)
    d("CB_V64_CANON_NAN", V64_CANON_NAN, True)
    out.append("")
    for k, v in TAGS.items():
        d(f"CB_T_{k}", v)
    out.append("")
    for k, v in OPS.items():
        d(f"CB_OP_{k}", v)
    d("CB_N_OPS", len(OPS))
    for k, v in HIER_RELS.items():
        d(f"CB_HIER_{k.upper()}", v)
    for k, v in TS_FIELDS.items():
        d(f"CB_TS_{k.upper()}", v)
    for k, v in TYPE_CODES.items():
        d("CB_TYPE_" + k.replace("google.protobuf.", "").upper(), v)
    out.append("")
    d("CB_FLAT_DNF", FLAT_DNF)
    for k, v in TERM_OPS.items():
        d(f"CB_TERM_{k}", v)
    d("CB_TERM_CI_MASK", TERM_CI_MASK, True)
    d("CB_TERM_LIT_F", TERM_LIT_F, True)
    d("CB_TERM_GROUP_END", TERM_GROUP_END, True)
    for k, v in OPK.items():
        d(f"CB_OPK_{k}", v)
    d("CB_FLAT_NOT_FAST", FLAT_NOT_FAST, True)
    d("CB_LOOP_ALL", LOOP_ALL)
    d("CB_LOOP_EXISTS", LOOP_EXISTS)
    d("CB_LOOP_EXISTS_ONE", LOOP_EXISTS_ONE)
    d("CB_LOOP_MAP", LOOP_MAP)
    d("CB_LOOP_FILTER", LOOP_FILTER)
    d("CB_LOOP_TMAP", LOOP_TMAP)
    d("CB_LOOP_TENTRY", LOOP_TENTRY)
    d("CB_LOOP_SORTBY", LOOP_SORTBY)
    for k, v in FNS.items():
        d(f"CB_FN_{k}", v)
    d("CB_MAX_STACK", MAX_STACK)
    d("CB_MAX_LOOP_DEPTH", MAX_LOOP_DEPTH)
    d("CB_MAX_VARS", MAX_VARS)
    d("CB_MAX_CHAIN", MAX_CHAIN)
    d("CB_MAX_ROLE_COLS", MAX_ROLE_COLS)
    d("CB_MAX_CLASS_PATS", MAX_CLASS_PATS)
    d("CB_BATCH_FLAG_LENIENT", BATCH_FLAG_LENIENT)
    d("CB_FORMAT_ARGS_STACK", FORMAT_ARGS_STACK)
    d("CB_FORMAT_ARGS_LIST", FORMAT_ARGS_LIST)
    d("CB_FMT_PREC_DEFAULT", FMT_PREC_DEFAULT, True)
    for k, v in META_SRC.items():
        d(f"CB_META_SRC_{k}", v)
    d("CB_IMAGE_SECTIONS", IMAGE_SECTIONS)
    d("CB_OUT_UNLOWERED_ACTIVATED", OUT_UNLOWERED_ACTIVATED)
    d("CB_OUT_UNLOWERED_NOT_MET", OUT_UNLOWERED_NOT_MET)
    for k, v in OUT_TAGS.items():
        d(f"CB_OUT_{k}", v)
    d("CB_OUT_RECORD_HEADER", OUT_RECORD_HEADER)
    d("CB_OUT_ENTRY_HEADER", OUT_ENTRY_HEADER)
    d("CB_OUT_MAX_STACK", OUT_MAX_STACK)
    d("CB_OUT_MAX_DEPTH", OUT_MAX_DEPTH)
    out.append("")
    out.append("""typedef struct { uint32_t magic, version, n_sections, flags; uint64_t total_bytes, reserved; } cb_blob_header;
typedef struct { uint32_t id, elem_bytes; uint64_t offset, n_bytes; } cb_section_desc;
typedef struct { uint32_t row_start, n_rows, cond_base, n_conds; } cb_block;
typedef struct { uint16_t role, cond, drcond, respat; uint8_t effect, flags; uint16_t n_pats; uint32_t pat_start; } cb_row;
typedef struct { uint32_t code_off, code_len, flat_off, flat_info; } cb_cond;
typedef struct { uint8_t op, a; uint16_t b; uint32_t c; } cb_instr;
typedef struct { uint8_t op, flags, xk, yk; uint32_t x, y; uint16_t xa, ya; } cb_term;   /* 16 B = two CODE slots */
typedef struct { uint32_t tag, pad; uint64_t bits; } cb_const;
typedef struct { uint32_t role, rule_start, n_rules, pad; } cb_rolepol_entry;
typedef struct { uint32_t respat, cond, apat_start, n_apats; } cb_rolepol_rule;
/* decision metadata plane (cgpu_check_meta): per (request, action) one word -- scope id of the deciding scope (0xFFFF: none) |
 * source << 16 | role id << 24 (source CB_META_SRC_ROLE_POLICY) -- and per request the first scope of each chain + the
 * effective derived roles as a bit set over MANIFEST.derived_roles */
typedef struct { uint16_t principal_first_scope, resource_first_scope; uint32_t flags; uint64_t effective_derived_roles; } cb_request_meta;
/* rule outputs (cgpu_check_outputs): an OUT_ENTRIES record, and the head of every request's output record */
typedef struct { uint32_t src, activated, not_met, flags; } cb_out_entry;
typedef struct { uint32_t bytes_needed, n_entries; } cb_out_record;
/* request header columns (SURVEY.md 8(d): 24 B / request) */
typedef struct { uint32_t principal_id, kind_class, resource_scope, principal_scope; } cb_hdr0;   /* 16 B */
typedef struct { uint16_t resource_version, principal_version; uint32_t action_set_id; } cb_hdr1;  /*  8 B */
""")
    out.append("#endif")
    return "\n".join(out) + "\n"


if __name__ == "__main__":
    import os
    root = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    path = os.path.join(root, "include", "cerbos_b200_format.h")
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        f.write(c_header())
    print("wrote", path)
