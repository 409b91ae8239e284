"""RuleTable -> flattened, HBM-resident table blob (host side, once per policy change).

H100-first replacement for the reference's in-memory index
(``index.Impl.IndexRules`` internal/ruletable/index/index.go:353-437, the five
inverted indexes of mem.go:57-220, ``indexRules`` internal/ruletable/ruletable.go:563-601,
``compileParentRoleAncestors`` index.go:842-881): instead of hash-map row sets that
are intersected per request, rows are grouped into *blocks* addressed by dense
integer keys so that the kernel finds every candidate row with one table lookup:

  resource block   (version, resource pattern, scope)      rows of one resource policy
  principal block  (version, principal,        scope)      rows of one principal policy
  role policies    (version, scope) -> [(role, allow rules)]  for the DENY synthesis of
                                                              index.go:688-776
  scope tables     parent pointers + per-kind membership + scope permissions
                   (GetAllScopes ruletable.go:611-645, scopeScopePermissions :584-586)
  parent roles     transitive closure per (scope, role)    (index.go:805-881)

Strings (roles, actions, kinds, scopes, literals) become dictionary ids; action and
resource *globs* are resolved by the batch encoder against the pattern dictionaries
kept in the MANIFEST section.  Conditions become bytecode (bytecode.py).
"""
from __future__ import annotations

import json
import struct

import numpy as np

from ..policy import namer
from ..policy.globs import is_glob
from ..policy.model import KIND_PRINCIPAL, KIND_RESOURCE, RuleTable, SP_UNSPECIFIED
from . import layout as L
from .bytecode import TableBuilderCtx, Unsupported, compile_condition, compile_flat, compile_value, const_v64


class _Dict:
    def __init__(self):
        self.ids = {}
        self.items = []

    def add(self, s):
        i = self.ids.get(s)
        if i is None:
            i = len(self.items)
            self.ids[s] = i
            self.items.append(s)
        return i

    def __len__(self):
        return len(self.items)


class FlatTable:
    """Result of flatten(): the blob plus host-side views used by the encoder and tests."""

    def __init__(self, blob: bytes, manifest: dict, sections: dict):
        self.blob = blob
        self.manifest = manifest
        self.sections = sections  # name -> numpy array (host copies)


def _scope_ancestors(scope: str):
    return namer.scope_parents(scope)


def flatten(rt: RuleTable, globals_=None) -> FlatTable:
    ctx = TableBuilderCtx(globals_=globals_)
    versions, scopes, respats, principals, roles, apats = _Dict(), _Dict(), _Dict(), _Dict(), _Dict(), _Dict()

    rows = list(rt.rows)
    # ---- dictionaries -------------------------------------------------------------------------------
    for r in rows:
        versions.add(r.version)
        scopes.add(r.scope)
        respats.add(r.resource)
        if r.policy_kind == KIND_PRINCIPAL:
            principals.add(r.principal)
        if r.role and r.role != "*":
            roles.add(r.role)
        if r.action is not None and not r.allow_actions:
            apats.add(r.action)
        for a in r.allow_actions or []:
            apats.add(a)
    for scope, rmap in rt.scope_parent_roles.items():
        for role, parents in rmap.items():
            roles.add(role)
            for p in parents:
                roles.add(p)
    for drs in rt.policy_derived_roles.values():
        for dr in drs.values():
            for pr in dr.parent_roles:
                if pr != "*":
                    roles.add(pr)
    dr_names = sorted({name for drs in rt.policy_derived_roles.values() for name in drs})
    if len(dr_names) > 64:
        raise Unsupported(f"more than 64 derived role names ({len(dr_names)})")
    dr_name_ix = {nm: i for i, nm in enumerate(dr_names)}
    for name, lim in (("roles", len(roles)), ("action patterns", len(apats)), ("resource patterns", len(respats))):
        if lim >= 0xFFFF:
            raise Unsupported(f"too many {name} ({lim})")
    nV, nS, nRP, nP, nR, nAP = len(versions), len(scopes), len(respats), len(principals), len(roles), len(apats)
    if nV * max(nRP, 1) * max(nS, 1) > (1 << 26):
        raise Unsupported("resource block map too large for the dense layout")

    # ---- scope tables ---------------------------------------------------------------------------------
    scope_parent = np.full(max(nS, 1), L.NONE32, dtype=np.uint32)
    scope_flags = np.zeros(max(nS, 1), dtype=np.uint32)
    max_depth = 1
    for s, sid in scopes.ids.items():
        for anc in _scope_ancestors(s):
            if anc in scopes.ids:
                scope_parent[sid] = scopes.ids[anc]
                break
    for sid in range(nS):
        d, cur = 1, sid
        while scope_parent[cur] != L.NONE32:
            cur = int(scope_parent[cur])
            d += 1
        max_depth = max(max_depth, d)
    if max_depth > L.MAX_CHAIN:
        raise Unsupported(f"scope chain deeper than {L.MAX_CHAIN}")
    perms = {}
    for r in rows:
        sid = scopes.ids[r.scope]
        scope_flags[sid] |= L.SCOPE_FLAG_PRINCIPAL if r.policy_kind == KIND_PRINCIPAL else L.SCOPE_FLAG_RESOURCE
        if r.scope_permissions != SP_UNSPECIFIED:
            perms[sid] = r.scope_permissions  # last writer wins (ruletable.go:584-586)
    for sid, p in perms.items():
        scope_flags[sid] |= p << L.SCOPE_PERM_SHIFT

    # ---- blocks + rows + conditions -----------------------------------------------------------------------
    res_block_map = np.full(max(nV * nRP * nS, 1), L.NONE32, dtype=np.uint32)
    res_exists = np.zeros(max(nV * nRP * nS, 1), dtype=np.uint8)
    prin_block_map = np.full(max(nV * nP * nS, 1), L.NONE32, dtype=np.uint32)
    prin_exists = np.zeros(max(nV * nS, 1), dtype=np.uint8)

    groups: dict[tuple, list] = {}
    rolepol: dict[tuple, dict] = {}
    for r in rows:
        v, s, rp = versions.ids[r.version], scopes.ids[r.scope], respats.ids[r.resource]
        ridx = (v * nRP + rp) * nS + s
        res_exists[ridx] |= L.EXISTS_ANY_ROW
        if r.policy_kind == KIND_RESOURCE:
            res_exists[ridx] |= L.EXISTS_RESOURCE_KIND
        else:
            prin_exists[v * nS + s] = 1
        if r.from_role_policy:
            if r.allow_actions:
                rolepol.setdefault((v, s), {}).setdefault(r.role, []).append(r)
            continue
        key = ("P", v, principals.ids[r.principal], s) if r.policy_kind == KIND_PRINCIPAL else ("R", v, rp, s)
        groups.setdefault(key, [])
        if r.action is not None:
            groups[key].append(r)

    blocks, row_recs, conds, code, row_apats = [], [], [], [], []
    pending_outputs: list = []   # (row index, Row) of every row with a rule output, compiled after all conditions
    dr_off, dr_entries, dr_parents = [], [], []
    block_shapes: set = set()
    code_ix: dict[tuple, tuple] = {}

    def add_program(cond, params) -> int:
        """Compiles and appends to CONDS; returns the global cond id."""
        prog = compile_condition(ctx, cond, params)

        def put(instrs):
            k = tuple(tuple(i) for i in instrs)
            ent = code_ix.get(k)
            if ent is None:
                ent = (len(code), len(instrs))
                code_ix[k] = ent
                code.extend(instrs)
            return ent

        gen = put(prog)
        flat = compile_flat(ctx, cond, params)
        if flat is not None:
            negate, n_terms, words = flat
            fk = ("flat",) + tuple(tuple(i) for i in words)
            fent = code_ix.get(fk)
            if fent is None:
                if len(code) % 2:
                    code.append([L.OPS["RET"], 0, 0, 0])      # terms are 16 bytes: keep them 16-byte aligned
                fent = (len(code), len(words))
                code_ix[fk] = fent
                code.extend(words)
            foff = fent[0]
            conds.append((gen[0], gen[1], foff, n_terms | (L.FLAT_DNF << 16) | (negate << 24)))
        else:
            conds.append((gen[0], gen[1], 0, 0))
        return len(conds) - 1

    for key, grows in groups.items():
        kind, v, ent, s = key
        bid = len(blocks)
        if kind == "P":
            prin_block_map[(v * nP + ent) * nS + s] = bid
        else:
            res_block_map[(v * nRP + ent) * nS + s] = bid
        cond_base = len(conds)
        local: dict[tuple, int] = {}

        def local_cond(cond, params):
            if cond is None:
                return 0
            k = (id(cond), id(params) if params is not None else 0)
            li = local.get(k)
            if li is None:
                gid = add_program(cond, params)
                li = gid - cond_base + 1
                local[k] = li
            if li >= 0xFFFF:
                raise Unsupported("too many conditions in one policy")
            return li

        row_start = len(row_recs)
        # rows that differ only in their action pattern are merged into one row with a pattern list -- except in a block
        # with rule outputs, where every rule action stays a row of its own in the reference's order: outputs are emitted
        # per visited row, and a merged row could move a DENY ahead of an output row
        with_outputs = any(r.emit_activated is not None or r.emit_not_met is not None for r in grows)
        merged: dict[tuple, list] = {}
        out_rows: list = []
        for r in grows:
            try:
                c_ix, dc_ix = local_cond(r.condition, r.params), local_cond(r.dr_condition, r.dr_params)
            except Unsupported as e:     # name the policy (and rule / derived role) the construct came from
                where = r.origin_fqn or "?"
                if getattr(r, "name", ""):
                    where += f" rule {r.name!r}"
                if r.origin_derived_role:
                    where += f" (derived role {r.origin_derived_role!r})"
                raise Unsupported(f"{where}: {e}") from e
            key2 = (L.ROLE_ANY if r.role == "*" else roles.ids[r.role], c_ix, dc_ix,
                    respats.ids[r.resource] if kind == "P" else L.NONE16, r.effect,
                    L.ROW_FLAG_PRINCIPAL if kind == "P" else 0)
            ap = apats.ids[r.action]
            if with_outputs:
                out_rows.append((key2, [ap]))
                if r.emit_activated is not None or r.emit_not_met is not None:
                    pending_outputs.append((row_start + len(out_rows) - 1, r))
                continue
            pats = merged.setdefault(key2, [])
            if ap not in pats:
                pats.append(ap)
        block_rows = out_rows if with_outputs else list(merged.items())
        for key2, pats in block_rows:
            if len(pats) > 0xFFFF:
                raise Unsupported("too many action patterns on one rule")
            row_recs.append(key2 + (len(pats), len(row_apats)))
            row_apats.extend(pats)
        blocks.append((row_start, len(row_recs) - row_start, cond_base, len(conds) - cond_base))
        # shape of the block = everything that steers the kernel's control flow through it
        block_shapes.add((tuple(k2[:3] + k2[4:] + (tuple(p),) for k2, p in block_rows), tuple(conds[cond_base:])))
        # derived roles of this resource policy (evaluated once per scope for effectiveDerivedRoles, ruletable.go:936-979);
        # the reference looks them up under the request's own kind, so only exact-name policies carry any
        dr_off.append(len(dr_entries))
        if kind == "R" and not is_glob(respats.items[ent]):
            fqn = namer.resource_policy_fqn(respats.items[ent], versions.items[v], scopes.items[s])
            for nm, dr in sorted((rt.policy_derived_roles.get(fqn) or {}).items()):
                cid = 0 if dr.condition is None else add_program(dr.condition, dr.params) + 1
                dr_entries.append((dr_name_ix[nm], cid, len(dr_parents), len(dr.parent_roles)))
                dr_parents.extend(L.ROLE_ANY if pr == "*" else roles.ids[pr] for pr in dr.parent_roles)

    # ---- role policies ----------------------------------------------------------------------------------------
    rp_off = np.zeros(nV * nS + 1, dtype=np.uint32)
    rp_entries, rp_rules, rp_apats = [], [], []
    for v in range(nV):
        for s in range(nS):
            rp_off[v * nS + s] = len(rp_entries)
            for role, rrows in (rolepol.get((v, s)) or {}).items():
                rule_start = len(rp_rules)
                for r in rrows:
                    cid = 0
                    if r.condition is not None:
                        try:
                            cid = add_program(r.condition, None) + 1
                        except Unsupported as e:
                            raise Unsupported(f"{r.origin_fqn or '?'}: {e}") from e
                    rp_rules.append((respats.ids[r.resource], cid, len(rp_apats), len(r.allow_actions)))
                    rp_apats.extend(apats.ids[a] for a in r.allow_actions)
                rp_entries.append((roles.ids[role], rule_start, len(rp_rules) - rule_start, 0))
    rp_off[nV * nS] = len(rp_entries)

    # ---- parent roles (transitive closure per scope; index.go:842-881) ------------------------------------------
    has_parents = any(parents for rmap in rt.scope_parent_roles.values() for parents in rmap.values())
    par_off = np.zeros(nS * nR + 1, dtype=np.uint32)
    par_list = []
    if has_parents:
        def collect(scope, role, acc, visited):
            if role in visited:
                return
            visited.add(role)
            for pr in rt.scope_parent_roles.get(scope, {}).get(role, []):
                if pr not in acc:
                    acc.append(pr)
                collect(scope, pr, acc, visited)
        for s_name, sid in scopes.ids.items():
            for role, rid in roles.ids.items():
                pass
        for sid in range(nS):
            s_name = scopes.items[sid]
            for rid in range(nR):
                par_off[sid * nR + rid] = len(par_list)
                if s_name in rt.scope_parent_roles and roles.items[rid] in rt.scope_parent_roles[s_name]:
                    acc = []
                    collect(s_name, roles.items[rid], acc, set())
                    par_list.extend(roles.ids[p] for p in acc)
        par_off[nS * nR] = len(par_list)

    # ---- rule outputs (after every condition, so that a table's slots, constants and code offsets keep their numbers) -----
    # An expression the device cannot lower leaves its entry unlowered: the table still builds, and only a request that
    # visits the row fails (CGPU_ERR_UNSUPPORTED).
    row_out = np.full(max(len(row_recs), 1), L.NONE32, dtype=np.uint32)
    out_entries, out_srcs, unlowered = [], _Dict(), []

    def add_output(expr, params):
        try:
            prog = compile_value(ctx, expr, params)
        except Unsupported as e:
            return None, str(e)
        ent = code_ix.get(tuple(tuple(i) for i in prog))
        if ent is None:
            ent = (len(code), len(prog))
            code_ix[tuple(tuple(i) for i in prog)] = ent
            code.extend(prog)
        return ent[0], ""

    for rix, r in pending_outputs:
        src = f"{namer.policy_key_from_fqn(r.origin_fqn)}#{r.name}"
        offs, flags = [L.NONE32, L.NONE32], 0
        for w, (expr, bit, when) in enumerate(((r.emit_activated, L.OUT_UNLOWERED_ACTIVATED, "ruleActivated"),
                                              (r.emit_not_met, L.OUT_UNLOWERED_NOT_MET, "conditionNotMet"))):
            if expr is None:
                continue
            off, why = add_output(expr, r.params)
            if off is None:
                flags |= bit
                unlowered.append({"policy": namer.policy_key_from_fqn(r.origin_fqn), "rule": r.name, "kind": r.resource,
                                  "when": when, "reason": why})
            else:
                offs[w] = off
        row_out[rix] = len(out_entries)
        out_entries.append((out_srcs.add(src), offs[0], offs[1], flags))

    # ---- strings: everything the kernels may compare against request strings ---------------------------------------
    # principals must be table strings so that hdr.principal_id (a string id) can be mapped to a principal index
    prin_str = [ctx.strings.intern(p) for p in principals.items]
    dr_name_str = [ctx.strings.intern(nm) for nm in dr_names]
    n_strings = len(ctx.strings)
    prin_of_string = np.full(max(n_strings, 1), L.NONE32, dtype=np.uint32)
    for pi, sid in enumerate(prin_str):
        prin_of_string[sid] = pi
    str_off = np.zeros(n_strings + 1, dtype=np.uint32)
    chunks = []
    pos = 0
    for i, s in enumerate(ctx.strings.items):
        b = s.encode("utf-8")
        str_off[i] = pos
        chunks.append(b)
        pos += len(b)
    str_off[n_strings] = pos
    str_bytes = np.frombuffer(b"".join(chunks) + b"\0" * 16, dtype=np.uint8)

    # ---- assemble -------------------------------------------------------------------------------------------------------
    meta = np.zeros(L.META_WORDS, dtype=np.uint32)
    for k, val in dict(
        n_versions=nV, n_respats=nRP, n_scopes=nS, n_principals=nP, n_roles=nR, n_apats=nAP,
        n_blocks=len(blocks), n_rows=len(row_recs), n_conds=len(conds), n_code=len(code), n_consts=len(ctx.consts),
        n_slots=len(ctx.slots), n_strings=n_strings, has_role_policies=int(bool(rp_entries)),
        has_parent_roles=int(has_parents), has_principal_policies=int(nP > 0), max_stack=ctx.max_stack,
        max_loop_depth=ctx.max_loop_depth, n_vars=ctx.n_vars, theap_words=len(ctx.theap),
        uses_pid=int(ctx.uses_pid), uses_now=int(ctx.uses_now), max_scope_depth=max_depth,
        direct_kinds=int(not any(is_glob(p) for p in respats.items)), block_shapes=len(block_shapes),
        uses_runtime=int(ctx.uses_runtime), n_dr_names=len(dr_names), n_output_rows=len(out_entries),
        n_unlowered_outputs=len(unlowered),
    ).items():
        meta[L.META[k]] = val

    blocks_a = np.array(blocks or [(0, 0, 0, 0)], dtype=np.uint32).reshape(-1, 4)
    rows_a = np.zeros(max(len(row_recs), 1), dtype=np.dtype([
        ("role", "<u2"), ("cond", "<u2"), ("drcond", "<u2"), ("respat", "<u2"),
        ("effect", "u1"), ("flags", "u1"), ("n_pats", "<u2"), ("pat_start", "<u4")]))
    for i, rec in enumerate(row_recs):
        rows_a[i] = rec
    # slots read by the conditions of each block (prefetch list for the kernel)
    slot_ops_c = {L.OPS["SLOT"], L.OPS["HAS_SLOT"]}
    slot_ops_b = {L.OPS["CMP_SLOT_CONST"], L.OPS["CMP_SLOT_SLOT"], L.OPS["CMP_SLOT_PID"], L.OPS["IN_SLOT_CONST"],
                  L.OPS["IN_CONST_SLOT"]}
    bs_off = np.zeros(len(blocks) + 1, dtype=np.uint32)
    bs_list = []
    for bi, (_rs, _nr, cbase, ncond) in enumerate(blocks):
        bs_off[bi] = len(bs_list)
        seen = []
        for ci in range(cbase, cbase + ncond):
            coff, clen, foff, finfo = conds[ci]
            if finfo:
                for q in range(finfo & 0xFFFF):
                    w0, w1 = code[foff + 2 * q], code[foff + 2 * q + 1]
                    xk, yk = w0[2] & 0xFF, w0[2] >> 8
                    yv = w1[0] | (w1[1] << 8) | (w1[2] << 16)
                    for kind_, v_ in ((xk, w0[3]), (yk, yv)):
                        if kind_ in (L.OPK["SLOT"], L.OPK["SLOT_ELEM"], L.OPK["SLOT_SIZE"]) and v_ not in seen:
                            seen.append(v_)
                continue
            spans = [(coff, clen)]
            for off, ln in spans:
                for ins in code[off:off + ln]:
                    if ins[0] in slot_ops_c and ins[3] not in seen:
                        seen.append(ins[3])
                    if ins[0] in slot_ops_b and ins[2] not in seen:
                        seen.append(ins[2])
                    if ins[0] == L.OPS["CMP_SLOT_SLOT"] and ins[3] not in seen:
                        seen.append(ins[3])
        bs_list.extend(seen)
    bs_off[len(blocks)] = len(bs_list)
    conds_a = np.array(conds or [(0, 0, 0, 0)], dtype=np.uint32).reshape(-1, 4)
    code_a = np.zeros(max(len(code), 1), dtype=np.dtype([("op", "u1"), ("a", "u1"), ("b", "<u2"), ("c", "<u4")]))
    for i, ins in enumerate(code):
        code_a[i] = tuple(ins)
    consts_a = np.zeros(max(len(ctx.consts), 1), dtype=np.dtype([("tag", "<u4"), ("pad", "<u4"), ("bits", "<u8")]))
    for i, cv in enumerate(ctx.consts):
        consts_a[i] = (cv.tag, 0, cv.bits)
    theap_a = np.array(ctx.theap or [0], dtype=np.uint64)
    consts_v64_a = np.array([const_v64(ctx, cv) for cv in ctx.consts] or [0], dtype=np.uint64)

    manifest = {
        "versions": versions.items, "scopes": scopes.items, "respats": respats.items, "principals": principals.items,
        "roles": roles.items, "apats": apats.items,
        "slots": [list(p) for p, _ in sorted(ctx.slots.items(), key=lambda kv: kv[1])],
        "strings": ctx.strings.items,
        "scope_flags": [int(x) for x in scope_flags[:nS]],
        "scope_parent": [int(x) for x in scope_parent[:nS]],
        "parent_role_scopes": sorted(s for s, rmap in rt.scope_parent_roles.items() if any(rmap.values())),
        "row_pat_start": [int(r[7]) for r in row_recs], "row_apats": [int(x) for x in row_apats],
        "derived_roles": dr_names,
    }
    if out_entries:
        manifest["output_sources"] = out_srcs.items
        manifest["unlowered_outputs"] = unlowered
    man_bytes = json.dumps(manifest, ensure_ascii=False, separators=(",", ":")).encode("utf-8")

    secs = [
        ("META", meta, 4), ("SCOPE_PARENT", scope_parent, 4), ("SCOPE_FLAGS", scope_flags, 4),
        ("RES_BLOCK_MAP", res_block_map, 4), ("RES_EXISTS", res_exists, 1),
        ("PRIN_BLOCK_MAP", prin_block_map, 4), ("PRIN_EXISTS", prin_exists, 1),
        ("PRIN_OF_STRING", prin_of_string, 4), ("BLOCKS", blocks_a, 16), ("ROWS", rows_a, 16),
        ("CONDS", conds_a, 16), ("CODE", code_a, 8), ("CONSTS", consts_a, 16), ("THEAP", theap_a, 8),
        ("STR_OFF", str_off, 4), ("STR_BYTES", str_bytes, 1),
        ("ROLE_PARENTS_OFF", par_off, 4), ("ROLE_PARENTS", np.array(par_list or [0], dtype=np.uint32), 4),
        ("ROLEPOL_OFF", rp_off, 4),
        ("ROLEPOL_ENTRIES", np.array(rp_entries or [(0, 0, 0, 0)], dtype=np.uint32).reshape(-1, 4), 16),
        ("ROLEPOL_RULES", np.array(rp_rules or [(0, 0, 0, 0)], dtype=np.uint32).reshape(-1, 4), 16),
        ("ROLEPOL_APATS", np.array(rp_apats or [0], dtype=np.uint32), 4),
        ("CONSTS_V64", consts_v64_a, 8),
        ("ROW_APATS", np.array(row_apats or [0], dtype=np.uint32), 4),
        ("BLOCK_SLOTS_OFF", bs_off, 4), ("BLOCK_SLOTS", np.array(bs_list or [0], dtype=np.uint32), 4),
        ("DR_OFF", np.array(dr_off + [len(dr_entries)], dtype=np.uint32), 4),
        ("DR_ENTRIES", np.array(dr_entries or [(0, 0, 0, 0)], dtype=np.uint32).reshape(-1, 4), 16),
        ("DR_PARENTS", np.array(dr_parents or [0], dtype=np.uint32), 4),
        ("DR_NAME_STR", np.array(dr_name_str or [0], dtype=np.uint32), 4),
    ]
    if out_entries:
        secs += [("ROW_OUT", row_out, 4), ("OUT_ENTRIES", np.array(out_entries, dtype=np.uint32).reshape(-1, 4), 16)]
    secs.append(("MANIFEST", np.frombuffer(man_bytes, dtype=np.uint8), 1))
    assert rows_a.dtype.itemsize == 16 and code_a.dtype.itemsize == 8 and consts_a.dtype.itemsize == 16

    hdr_bytes = 32 + 24 * len(secs)
    off = (hdr_bytes + L.ALIGN - 1) // L.ALIGN * L.ALIGN
    descs, payload = [], []
    for name, arr, eb in secs:
        raw = np.ascontiguousarray(arr).tobytes()
        descs.append((L.SECTIONS[name], eb, off, len(raw)))
        padded = (len(raw) + L.ALIGN - 1) // L.ALIGN * L.ALIGN
        payload.append(raw + b"\0" * (padded - len(raw)))
        off += padded
    total = off
    out = bytearray()
    out += struct.pack("<IIIIQQ", L.MAGIC, L.VERSION, len(secs), 0, total, 0)
    for d in descs:
        out += struct.pack("<IIQQ", *d)
    out += b"\0" * ((hdr_bytes + L.ALIGN - 1) // L.ALIGN * L.ALIGN - len(out))
    for p in payload:
        out += p
    assert len(out) == total
    return FlatTable(bytes(out), manifest, {name: arr for name, arr, _ in secs})
