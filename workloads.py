"""Synthetic CheckResources workloads C1..C3 (SURVEY.md 8(d), BASELINE.json `configs`).

Every workload provides
  * ``policies()``            policy documents (dicts, same shape as the reference's YAML),
  * ``fields(n)``             per-request logical fields as numpy arrays, drawn from SplitMix64
                              streams (seed 0xCE4B05 + cfg#, stream index = request index),
  * ``inputs(fields, idx)``   CheckInput dicts for a subset (what the reference's Go harness or the
                              Python oracle would be handed), and
  * ``columns(fields, enc)``  the same requests encoded directly (vectorised) into the SoA batch
                              columns of cerbos_b200/encode.py -- used for the 2^20 .. 2^24 batches
                              where a per-request Python encoder would take minutes.
tests/test_workloads.py checks that both routes give identical decisions.
"""
from __future__ import annotations

import numpy as np

from cerbos_b200.encode import Batch, Encoder, passes_for
from cerbos_b200.table import layout as L

SEED_BASE = 0xCE4B05
_GOLDEN = np.uint64(0x9E3779B97F4A7C15)
_DRAWS = 32  # draws reserved per request


import threading

_TLS = threading.local()  # .start: first request index of the window being generated (set by fields(n, start)); per thread


def splitmix(seed: int, n: int, draw: int) -> np.ndarray:
    """draw-th SplitMix64 output of the stream of every request start..start+n-1 (start: see fields(n, start))."""
    with np.errstate(over="ignore"):
        idx = (np.arange(n, dtype=np.uint64) + np.uint64(getattr(_TLS, 'start', 0))) * np.uint64(_DRAWS) + np.uint64(draw + 1)
        z = np.uint64(seed) + idx * _GOLDEN
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def _uniform(seed, n, draw, k):
    return (splitmix(seed, n, draw) % np.uint64(k)).astype(np.int64)


def _prob(seed, n, draw, p):
    return (splitmix(seed, n, draw) >> np.uint64(11)).astype(np.float64) * (1.0 / (1 << 53)) < p


def _box(tag, payload):
    return (np.uint64((L.V64_BOX_BASE | tag) << 48)) | payload.astype(np.uint64)


def _str_ids(enc: Encoder, strings):
    """Assigns ids the way the encoder would: table strings keep their table id, the rest are
    appended to the batch string table. Returns (ids array, batch string list)."""
    nts = enc.n_table_strings
    ids, extra, seen = [], [], {}
    for s in strings:
        i = enc.table_strings.get(s)
        if i is None:
            i = seen.get(s)
            if i is None:
                i = nts + len(extra)
                seen[s] = i
                extra.append(s.encode("utf-8"))
        ids.append(i)
    return np.array(ids, dtype=np.uint64), extra


def _kind_classes(enc: Encoder, kinds):
    """-> (hdr kind_class value per kind, CSR class list) using the encoder's direct / CSR encoding."""
    classes, class_list, vals = {}, [], []
    for k in kinds:
        vals.append(enc.kind_class(enc.kind_patterns(k), classes, class_list))
    return np.array(vals, dtype=np.uint32), class_list


def _finish_batch(enc: Encoder, n, hdr0, hdr1, roles, slots, heap, bstr_list, class_list, aset_list, max_actions):
    role_cols = roles.shape[0]
    class_off = np.zeros(len(class_list) + 1, dtype=np.uint32)
    cp = []
    for c, pats in enumerate(class_list):
        class_off[c] = len(cp)
        cp.extend(pats)
    class_off[len(class_list)] = len(cp)
    aset_k, aset_spread, row_am = enc.build_action_sets(aset_list, role_cols, max_actions)
    off = np.zeros(len(bstr_list) + 1, dtype=np.uint32)
    pos = 0
    for j, b in enumerate(bstr_list):
        off[j] = pos
        pos += len(b)
    off[len(bstr_list)] = pos
    bbytes = np.frombuffer(b"".join(bstr_list) + b"\0" * 16, dtype=np.uint8)
    kc, n_pass = passes_for(max_actions, role_cols)
    cols = [hdr0, hdr1, roles, slots, heap, off, bbytes, class_off, np.array(cp or [0], dtype=np.uint32),
            aset_k, aset_spread, row_am]
    return Batch(n, max_actions, role_cols, cols, None, n_pass, kc)


# =========================================================================================== C1
class C1:
    """hack/loadtest-shaped: 1 resource policy, 3 actions, role-only rules, 32x32 = 1024 pairs."""
    name = "C1"
    cfg = 1
    actions = ["view", "edit", "delete"]
    role_names = ["user", "editor", "admin", "guest"]
    default_n = 1024
    role_cols = 2
    n_slots = 0
    heap_bytes = 0

    def policies(self):
        return [{"apiVersion": "api.cerbos.dev/v1", "resourcePolicy": {
            "resource": "document", "version": "default", "rules": [
                {"actions": ["view"], "effect": "EFFECT_ALLOW", "roles": ["user", "admin"]},
                {"actions": ["edit"], "effect": "EFFECT_ALLOW", "roles": ["editor", "admin"]},
                {"actions": ["delete"], "effect": "EFFECT_ALLOW", "roles": ["admin"]},
            ]}}]

    def fields(self, n=None, start=0):
        n = n or self.default_n
        seed = SEED_BASE + self.cfg
        pr = (np.arange(n) + start) // 32 % 32      # principal index, materialised flat (one row per pair)
        rs = (np.arange(n) + start) % 32
        # roles are a property of the principal: derive them from the principal's own stream
        r0 = _uniform(seed, 32, 0, 4)[pr]
        two = _prob(seed, 32, 1, 0.5)[pr]
        r1 = (r0 + 1 + _uniform(seed, 32, 2, 3)[pr]) % 4
        return {"n": n, "pr": pr, "rs": rs, "r0": r0, "r1": np.where(two, r1, -1)}

    def inputs(self, f, idx):
        out = []
        for i in idx:
            roles = [self.role_names[f["r0"][i]]] + ([self.role_names[f["r1"][i]]] if f["r1"][i] >= 0 else [])
            out.append({"requestId": str(i), "actions": list(self.actions),
                        "principal": {"id": f"user{f['pr'][i]}", "roles": roles},
                        "resource": {"kind": "document", "id": f"doc{f['rs'][i]}"}})
        return out

    def columns(self, f, enc: Encoder) -> Batch:
        n = f["n"]
        pid_ids, extra = _str_ids(enc, [f"user{i}" for i in range(32)])
        hdr0 = np.zeros((n, 4), dtype=np.uint32)
        hdr0[:, 0] = pid_ids[f["pr"]]
        kvals, class_list = _kind_classes(enc, ["document"])
        hdr0[:, 1] = kvals[0]
        hdr0[:, 2] = enc.resolve_scope("")
        hdr0[:, 3] = enc.resolve_scope("")
        hdr1 = np.zeros(n, dtype=np.dtype([("rv", "<u2"), ("pv", "<u2"), ("aset", "<u4")]))
        hdr1["rv"] = enc.version_ids.get("default", L.NONE16)
        hdr1["pv"] = hdr1["rv"]
        rmap = np.array([enc.role_ids.get(r, L.ROLE_UNKNOWN) for r in self.role_names] + [L.ROLE_PAD], dtype=np.uint32)
        roles = np.stack([rmap[f["r0"]], rmap[f["r1"]]]).astype(np.uint32)
        slots = np.zeros((1, n), dtype=np.uint64)
        return _finish_batch(enc, n, hdr0, hdr1, roles, slots, np.zeros(1, dtype=np.uint64), extra,
                             class_list, [tuple(self.actions)], 3)

    # SURVEY.md 8(d): 24 + 4R + 8A + S + ceil(K/8)
    def bytes_per_request(self):
        return 24 + 4 * 2 + 0 + 0 + 1


# =========================================================================================== C2
class C2:
    """10 resource policies x 8 actions, 2 derived roles with CEL on request.resource.attr; batch 2^20.
    This is the configuration BASELINE.json's metric is quoted on for one H100."""
    name = "C2"
    cfg = 2
    actions = [f"a{i}" for i in range(8)]
    role_names = ["user", "manager", "admin"]
    statuses = ["OPEN", "PENDING", "CLOSED", "ARCHIVED"]
    default_n = 1 << 20
    n_principals = 65536
    n_kinds = 10
    role_cols = 2

    def policies(self):
        docs = [{"apiVersion": "api.cerbos.dev/v1", "derivedRoles": {"name": "c2_roles", "definitions": [
            {"name": "owner", "parentRoles": ["user"],
             "condition": {"match": {"expr": "R.attr.owner == P.id"}}},
            {"name": "dept_manager", "parentRoles": ["manager"],
             "condition": {"match": {"expr": 'R.attr.dept == P.attr.dept && R.attr.status in ["OPEN","PENDING"]'}}},
        ]}}]
        for k in range(self.n_kinds):
            docs.append({"apiVersion": "api.cerbos.dev/v1", "resourcePolicy": {
                "resource": f"kind_{k}", "version": "default", "importDerivedRoles": ["c2_roles"], "rules": [
                    {"actions": ["a0", "a1", "a2"], "effect": "EFFECT_ALLOW", "roles": ["user"]},
                    {"actions": ["a3", "a4"], "effect": "EFFECT_ALLOW", "derivedRoles": ["owner"]},
                    {"actions": ["a5", "a6"], "effect": "EFFECT_ALLOW", "derivedRoles": ["dept_manager"]},
                    {"actions": ["a7"], "effect": "EFFECT_ALLOW", "roles": ["admin"]},
                    {"actions": ["*"], "effect": "EFFECT_DENY", "roles": ["*"],
                     "condition": {"match": {"expr": "R.attr.locked == true"}}},
                ]}})
        return docs

    def fields(self, n=None, start=0):
        """Requests [start, start+n) of the workload's stream."""
        n = n or self.default_n
        seed = SEED_BASE + self.cfg
        _TLS.start = start
        try:
            return self._fields(n, seed)
        finally:
            _TLS.start = 0

    def _fields(self, n, seed):
        pid = _uniform(seed, n, 1, self.n_principals)
        own_other = _uniform(seed, n, 5, self.n_principals)
        r0 = _uniform(seed, n, 2, 3)
        r1 = (r0 + 1 + _uniform(seed, n, 4, 2)) % 3
        return {
            "n": n,
            "kind": _uniform(seed, n, 0, self.n_kinds),
            "pid": pid,
            "r0": r0,
            "r1": np.where(_prob(seed, n, 3, 0.5), r1, -1),
            "owner": np.where(_prob(seed, n, 6, 0.25), pid, own_other),
            "pdept": _uniform(seed, n, 7, 16),
            "rdept": _uniform(seed, n, 8, 16),
            "status": _uniform(seed, n, 9, 4),
            "locked": _prob(seed, n, 10, 0.05),
        }

    def inputs(self, f, idx):
        out = []
        for i in idx:
            roles = [self.role_names[f["r0"][i]]] + ([self.role_names[f["r1"][i]]] if f["r1"][i] >= 0 else [])
            out.append({"requestId": str(i), "actions": list(self.actions),
                        "principal": {"id": f"p{f['pid'][i]}", "roles": roles, "attr": {"dept": f"d{f['pdept'][i]}"}},
                        "resource": {"kind": f"kind_{f['kind'][i]}", "id": f"r{i}", "attr": {
                            "owner": f"p{f['owner'][i]}", "dept": f"d{f['rdept'][i]}",
                            "status": self.statuses[f["status"][i]], "locked": bool(f["locked"][i])}}})
        return out

    def columns(self, f, enc: Encoder) -> Batch:
        n = f["n"]
        pid_ids, extra = _str_ids(enc, [f"p{i}" for i in range(self.n_principals)])
        nts = enc.n_table_strings
        dept_ids, e2 = _str_ids(enc, [f"d{i}" for i in range(16)])
        # continue numbering of batch strings after `extra`
        dept_ids = np.where(dept_ids >= nts, dept_ids + np.uint64(len(extra)), dept_ids)
        extra = extra + e2
        st_ids, e3 = _str_ids(enc, self.statuses)
        st_ids = np.where(st_ids >= nts, st_ids + np.uint64(len(extra)), st_ids)
        extra = extra + e3
        kvals, class_list = _kind_classes(enc, [f"kind_{k}" for k in range(self.n_kinds)])
        hdr0 = np.zeros((n, 4), dtype=np.uint32)
        hdr0[:, 0] = pid_ids[f["pid"]]
        hdr0[:, 1] = kvals[f["kind"]]
        hdr0[:, 2] = enc.resolve_scope("")
        hdr0[:, 3] = enc.resolve_scope("")
        hdr1 = np.zeros(n, dtype=np.dtype([("rv", "<u2"), ("pv", "<u2"), ("aset", "<u4")]))
        hdr1["rv"] = enc.version_ids.get("default", L.NONE16)
        hdr1["pv"] = hdr1["rv"]
        rmap = np.array([enc.role_ids.get(r, L.ROLE_UNKNOWN) for r in self.role_names] + [L.ROLE_PAD], dtype=np.uint32)
        roles = np.stack([rmap[f["r0"]], rmap[f["r1"]]]).astype(np.uint32)
        slots = np.zeros((max(len(enc.slots), 1), n), dtype=np.uint64)
        vals = {
            ("principal", "attr", "dept"): _box(L.V64_STRING, dept_ids[f["pdept"]]),
            ("resource", "attr", "owner"): _box(L.V64_STRING, pid_ids[f["owner"]]),
            ("resource", "attr", "dept"): _box(L.V64_STRING, dept_ids[f["rdept"]]),
            ("resource", "attr", "status"): _box(L.V64_STRING, st_ids[f["status"]]),
            ("resource", "attr", "locked"): _box(L.V64_BOOL, f["locked"].astype(np.uint64)),
        }
        for s, path in enumerate(enc.slots):
            slots[s] = vals[path]
        return _finish_batch(enc, n, hdr0, hdr1, roles, slots, np.zeros(1, dtype=np.uint64), extra,
                             class_list, [tuple(self.actions)], 8)

    def bytes_per_request(self):
        return 24 + 4 * 2 + 8 * 5 + 0 + 1   # = 73 (SURVEY.md 8(d))


# =========================================================================================== C3
def _ragged_lists(lengths: np.ndarray, elem_fn, head=None):
    """Builds heap words for one variable-length list per request: [len, e0, e1, ...].
    elem_fn(req_index_array, pos_array) -> uint64 element words. Returns (words, offsets).
    head: the first word of every record if it is not the number of elements (a map's [n, keys..., values...] has 2n)."""
    n = len(lengths)
    sizes = lengths + 1
    offs = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(sizes, out=offs[1:])
    words = np.zeros(offs[-1], dtype=np.uint64)
    words[offs[:-1]] = (lengths if head is None else head).astype(np.uint64)
    req = np.repeat(np.arange(n), lengths)
    pos = np.arange(lengths.sum()) - np.repeat(offs[:-1] - np.arange(n), lengths)
    words[np.repeat(offs[:-1] + 1, lengths) + pos] = elem_fn(req, pos)
    return words, offs[:-1]


class C3:
    """100 resource policies = 20 kinds x 5 scopes (3-level chain), 20 CEL conditions incl. string / list ops on
    principal.attr, REQUIRE_PARENTAL_CONSENT leaves; batch 2^24 (BASELINE.json configs[2])."""
    name = "C3"
    cfg = 3
    actions = [f"a{i}" for i in range(8)]
    role_names = ["user", "manager", "admin", "auditor"]
    scopes = ["", "t0", "t1", "t0.d0", "t1.d0"]
    req_scopes = ["", "t0", "t1", "t0.d0", "t1.d0", "t0.d9"]
    tiers = ["gold", "silver", "bronze", "banned"]
    regions = ["eu", "us", "apac", "latam"]
    default_n = 1 << 24
    n_kinds = 20
    n_principals = 65536
    role_cols = 3
    conditions = [
        'P.attr.email.endsWith("@corp.example")',
        'P.attr.name.startsWith(R.attr.prefix)',
        '"eng" in P.attr.groups',
        'hasIntersection(P.attr.groups, R.attr.allowed_groups)',
        'P.attr.groups.exists(g, g == R.attr.team)',
        'size(P.attr.groups) > 2',
        'P.attr.level >= R.attr.min_level',
        'P.attr.region in ["eu", "us"]',
        'P.attr.level > 5 ? R.attr.tier == "gold" : R.attr.public == true',
        'R.attr.owner == P.id',
        'R.attr.team in P.attr.groups',
        'P.attr.name.contains("an")',
        'R.attr.public == true || P.attr.level >= 8',
        '!(P.attr.region == "apac")',
        'P.attr.groups.all(g, g != "g13")',
        'R.attr.tier in ["gold", "silver"] && P.attr.level > 2',
        'size(R.attr.allowed_groups) >= 1 && P.attr.groups[0] in R.attr.allowed_groups',
        'has(R.attr.prefix) && R.attr.prefix != ""',
        'P.attr.email.contains("@") && R.attr.min_level <= 9',
        'isSubset(R.attr.allowed_groups, P.attr.groups)',
    ]
    groups = ["eng"] + [f"g{i}" for i in range(1, 32)]
    words = ["".join(chr(97 + (i * 7 + j * 3) % 26) for j in range(3 + i % 6)) + ("an" if i % 5 == 0 else "") for i in range(256)]

    def policies(self):
        docs = []
        for k in range(self.n_kinds):
            for si, sc in enumerate(self.scopes):
                rules = []
                for j in range(8):
                    cond = self.conditions[(k * 8 + j + si * 3) % 20]
                    role = self.role_names[(j + k + si) % 3]
                    rule = {"actions": [f"a{j}"], "effect": "EFFECT_ALLOW", "roles": [role, "admin"] if j % 4 == 3 else [role]}
                    if (j + si) % 4 != 0:       # every fourth rule is unconditional
                        rule["condition"] = {"match": {"expr": cond}}
                    rules.append(rule)
                rules.append({"actions": ["*"], "effect": "EFFECT_DENY", "roles": ["*"],
                              "condition": {"match": {"expr": 'R.attr.tier == "banned"'}}})
                rp = {"resource": f"kind_{k}", "version": "default", "rules": rules}
                if sc:
                    rp["scope"] = sc
                if sc.endswith(".d0"):
                    rp["scopePermissions"] = "SCOPE_PERMISSIONS_REQUIRE_PARENTAL_CONSENT_FOR_ALLOWS"
                docs.append({"apiVersion": "api.cerbos.dev/v1", "resourcePolicy": rp})
        return docs

    def fields(self, n=None, start=0):
        n = n or self.default_n
        seed = SEED_BASE + self.cfg
        _TLS.start = start
        try:
            pid = _uniform(seed, n, 1, self.n_principals)
            r0 = _uniform(seed, n, 2, 4)
            nr = 1 + _uniform(seed, n, 3, 3)
            sc = _uniform(seed, n, 4, 5)
            f = {
                "n": n, "kind": _uniform(seed, n, 0, self.n_kinds), "pid": pid,
                "r0": r0, "r1": np.where(nr >= 2, (r0 + 1) % 4, -1), "r2": np.where(nr >= 3, (r0 + 2) % 4, -1),
                "scope": np.where(_prob(seed, n, 5, 0.05), 5, sc),
                "email_w": _uniform(seed, n, 6, 256), "email_corp": _prob(seed, n, 7, 0.5),
                "name_w": _uniform(seed, n, 8, 256), "prefix_w": _uniform(seed, n, 9, 256),
                "prefix_same": _prob(seed, n, 10, 0.3), "prefix_len": 1 + _uniform(seed, n, 11, 3),
                "level": _uniform(seed, n, 12, 10), "min_level": _uniform(seed, n, 13, 10),
                "region": _uniform(seed, n, 14, 4), "tier": _uniform(seed, n, 15, 4),
                "public": _prob(seed, n, 16, 0.3), "team": _uniform(seed, n, 17, 32),
                "owner": np.where(_prob(seed, n, 18, 0.25), pid, _uniform(seed, n, 19, self.n_principals)),
                "n_groups": 1 + _uniform(seed, n, 20, 6), "g_seed": splitmix(seed, n, 21),
                "n_allowed": 1 + _uniform(seed, n, 22, 4), "a_seed": splitmix(seed, n, 23),
            }
            return f
        finally:
            _TLS.start = 0

    @staticmethod
    def _members(seedv, count, pos):
        """pos-th element of a `count`-element subset of 0..31 drawn from seed: distinct by construction
        (start + pos * odd step mod 32)."""
        start = (seedv & np.uint64(31)).astype(np.int64)
        step = (((seedv >> np.uint64(5)) & np.uint64(15)).astype(np.int64) * 2 + 1)
        return (start + pos * step) % 32

    def _prefix(self, f, i):
        w = self.words[f["name_w"][i]] if f["prefix_same"][i] else self.words[f["prefix_w"][i]]
        return w[: f["prefix_len"][i]]

    def inputs(self, f, idx):
        out = []
        for i in idx:
            roles = [self.role_names[f[k][i]] for k in ("r0", "r1", "r2") if f[k][i] >= 0]
            ng, na = int(f["n_groups"][i]), int(f["n_allowed"][i])
            gs = [self.groups[self._members(f["g_seed"][i:i + 1], ng, np.array([p]))[0]] for p in range(ng)]
            al = [self.groups[self._members(f["a_seed"][i:i + 1], na, np.array([p]))[0]] for p in range(na)]
            dom = "@corp.example" if f["email_corp"][i] else "@other.example"
            res = {"kind": f"kind_{f['kind'][i]}", "id": f"r{i}", "attr": {
                "prefix": self._prefix(f, i), "allowed_groups": al, "team": self.groups[f["team"][i]],
                "min_level": int(f["min_level"][i]), "tier": self.tiers[f["tier"][i]], "public": bool(f["public"][i]),
                "owner": f"p{f['owner'][i]}"}}
            sc = self.req_scopes[f["scope"][i]]
            if sc:
                res["scope"] = sc
            out.append({"requestId": str(i), "actions": list(self.actions),
                        "principal": {"id": f"p{f['pid'][i]}", "roles": roles, "attr": {
                            "email": self.words[f["email_w"][i]] + dom, "name": self.words[f["name_w"][i]],
                            "groups": gs, "level": int(f["level"][i]), "region": self.regions[f["region"][i]]}},
                        "resource": res})
        return out

    def columns(self, f, enc: Encoder) -> Batch:
        n = f["n"]
        nts = enc.n_table_strings
        extra: list = []

        def ids_for(strings):
            nonlocal extra
            ids, e = _str_ids(enc, strings)
            # _str_ids numbers new strings from nts; shift by what is already in `extra`, dedupe against it
            out = []
            pos = {b: j for j, b in enumerate(extra)}
            for s_, i_ in zip(strings, ids):
                if i_ < nts:
                    out.append(int(i_))
                else:
                    bkey = s_.encode("utf-8")
                    j = pos.get(bkey)
                    if j is None:
                        j = len(extra)
                        pos[bkey] = j
                        extra.append(bkey)
                    out.append(nts + j)
            return np.array(out, dtype=np.uint64)

        pid_ids = ids_for([f"p{i}" for i in range(self.n_principals)])
        email_ids = ids_for([w + d for d in ("@other.example", "@corp.example") for w in self.words]).reshape(2, 256)
        name_ids = ids_for(self.words)
        prefixes = sorted({w[:L_] for w in self.words for L_ in (1, 2, 3)})
        pre_ix = {p_: j for j, p_ in enumerate(prefixes)}
        pre_ids = ids_for(prefixes)
        group_ids = ids_for(self.groups)
        tier_ids, region_ids = ids_for(self.tiers), ids_for(self.regions)
        # prefix string per request
        wsel = np.where(f["prefix_same"], f["name_w"], f["prefix_w"])
        pre_tab = np.array([[pre_ix[self.words[w][:L_]] for L_ in (1, 2, 3)] for w in range(256)], dtype=np.int64)
        pre_req = pre_ids[pre_tab[wsel, f["prefix_len"] - 1]]

        kvals, class_list = _kind_classes(enc, [f"kind_{k}" for k in range(self.n_kinds)])
        hdr0 = np.zeros((n, 4), dtype=np.uint32)
        hdr0[:, 0] = pid_ids[f["pid"]]
        hdr0[:, 1] = kvals[f["kind"]]
        sc_ids = np.array([enc.resolve_scope(s_) for s_ in self.req_scopes], dtype=np.uint32)
        hdr0[:, 2] = sc_ids[f["scope"]]
        hdr0[:, 3] = enc.resolve_scope("")
        hdr1 = np.zeros(n, dtype=np.dtype([("rv", "<u2"), ("pv", "<u2"), ("aset", "<u4")]))
        hdr1["rv"] = enc.version_ids.get("default", L.NONE16)
        hdr1["pv"] = hdr1["rv"]
        rmap = np.array([enc.role_ids.get(r, L.ROLE_UNKNOWN) for r in self.role_names] + [L.ROLE_PAD], dtype=np.uint32)
        roles = np.stack([rmap[f["r0"]], rmap[f["r1"]], rmap[f["r2"]]]).astype(np.uint32)

        box_s = lambda ids: _box(L.V64_STRING, ids)   # noqa: E731
        g_words, g_off = _ragged_lists(f["n_groups"], lambda req, pos: box_s(group_ids[self._members(f["g_seed"][req], None, pos)]))
        a_words, a_off = _ragged_lists(f["n_allowed"], lambda req, pos: box_s(group_ids[self._members(f["a_seed"][req], None, pos)]))
        heap = np.concatenate([g_words, a_words])
        batch_bit = np.uint64(L.V64_HEAP_BATCH_BIT)
        vals = {
            ("principal", "attr", "email"): box_s(email_ids[f["email_corp"].astype(np.int64), f["email_w"]]),
            ("principal", "attr", "name"): box_s(name_ids[f["name_w"]]),
            ("principal", "attr", "groups"): _box(L.V64_LIST, g_off.astype(np.uint64) | batch_bit),
            ("principal", "attr", "level"): f["level"].astype(np.float64).view(np.uint64),
            ("principal", "attr", "region"): box_s(region_ids[f["region"]]),
            ("resource", "attr", "prefix"): box_s(pre_req),
            ("resource", "attr", "allowed_groups"): _box(L.V64_LIST, (a_off + len(g_words)).astype(np.uint64) | batch_bit),
            ("resource", "attr", "team"): box_s(group_ids[f["team"]]),
            ("resource", "attr", "min_level"): f["min_level"].astype(np.float64).view(np.uint64),
            ("resource", "attr", "tier"): box_s(tier_ids[f["tier"]]),
            ("resource", "attr", "public"): _box(L.V64_BOOL, f["public"].astype(np.uint64)),
            ("resource", "attr", "owner"): box_s(pid_ids[f["owner"]]),
        }
        slots = np.zeros((max(len(enc.slots), 1), n), dtype=np.uint64)
        for s_, path in enumerate(enc.slots):
            slots[s_] = vals[path]
        return _finish_batch(enc, n, hdr0, hdr1, roles, slots, heap, extra, class_list, [tuple(self.actions)], 8)

    def bytes_per_request(self):
        return 24 + 4 * 3 + 8 * 12 + 64 + 1   # = 197 (SURVEY.md 8(d))



class C5:
    """Adversarial (BASELINE.json configs[4]): 1000 resource policies = 200 kinds x 5 scopes, 8 actions each, deep CEL --
    nested all/any/none trees, ternaries, map indexing with a dynamic key, two-variable comprehensions over maps,
    JWT claims from auxData (list membership, `in ... .split(" ")`, `timestamp(claim) > now()`), variables that
    reference variables -- Zipf(1.1)-skewed resource kinds.  Parity-test configuration: requests go through the
    generic encoder (no vectorised column builder), sizes of a few thousand."""
    name = "C5"
    cfg = 5
    actions = [f"a{i}" for i in range(8)]
    role_names = ["user", "manager", "admin", "auditor"]
    scopes = ["", "t0", "t1", "t0.d0", "t1.d0"]
    req_scopes = ["", "t0", "t1", "t0.d0", "t1.d0", "t0.d9"]
    tiers = ["gold", "silver", "bronze"]
    n_kinds = 200
    default_n = 1 << 26
    role_cols = 4
    leafs = [
        'R.attr.meta.tags[P.attr.tier] in ["hot", "warm"]',
        'P.attr.grants.exists(k, v, k == R.kind && "write" in v)',
        '"svc" in request.aux_data.jwt.aud',
        '"deploy" in request.aux_data.jwt.scope.split(" ")',
        'timestamp(request.aux_data.jwt.exp_ts) > now()',
        'V.is_internal && V.senior',
        'P.attr.level > 5 ? R.attr.meta.owner == P.id : R.attr.public == true',
        'request.aux_data.jwt.tier == P.attr.tier',
        'R.attr.meta.region in P.attr.regions',
        'size(P.attr.regions) > 1 || request.aux_data.jwt.iss == "https://issuer.example"',
        'has(R.attr.meta.owner) && R.attr.meta.owner != ""',
        'P.attr.level >= R.attr.min_level',
    ]
    regions = ["eu", "us", "apac", "latam"]

    def _tree(self, k, j, si):
        """condition tree of rule j of policy (kind k, scope si): depth-3 nests every third rule"""
        L_ = self.leafs
        a, b, c, d = (L_[(k + j * 3 + si + q) % len(L_)] for q in range(4))
        if j % 3 == 0:
            return {"all": {"of": [{"any": {"of": [{"expr": a}, {"none": {"of": [{"expr": b}]}}]}}, {"none": {"of": [{"all": {"of": [{"expr": c}, {"expr": d}]}}]}}]}}
        if j % 3 == 1:
            return {"any": {"of": [{"expr": a}, {"all": {"of": [{"expr": b}, {"expr": c}]}}]}}
        return {"expr": a}

    def policies(self):
        docs = []
        for k in range(self.n_kinds):
            for si, sc in enumerate(self.scopes):
                rules = []
                for j in range(8):
                    rule = {"actions": [f"a{j}"], "effect": "EFFECT_ALLOW", "roles": [self.role_names[(j + k + si) % 4]]}
                    if (j + si + k) % 5 != 0:
                        rule["condition"] = {"match": self._tree(k, j, si)}
                    rules.append(rule)
                rules.append({"actions": ["*"], "effect": "EFFECT_DENY", "roles": ["*"],
                              "condition": {"match": {"expr": 'request.aux_data.jwt.tier == "banned"'}}})
                rp = {"resource": f"kind_{k}", "version": "default", "rules": rules,
                      "variables": {"local": {"is_internal": 'request.aux_data.jwt.iss == "https://issuer.example"',
                                              "senior": "V.is_internal && P.attr.level >= 7"}}}
                if sc:
                    rp["scope"] = sc
                if sc.endswith(".d0"):
                    rp["scopePermissions"] = "SCOPE_PERMISSIONS_REQUIRE_PARENTAL_CONSENT_FOR_ALLOWS"
                docs.append({"apiVersion": "api.cerbos.dev/v1", "resourcePolicy": rp})
        return docs

    def fields(self, n=None, start=0):
        n = n or 4096
        seed = SEED_BASE + self.cfg
        _TLS.start = start
        try:
            # Zipf(s = 1.1) over the kinds by inverse CDF on a uniform draw
            w = 1.0 / np.arange(1, self.n_kinds + 1) ** 1.1
            cdf = np.cumsum(w) / w.sum()
            u = (splitmix(seed, n, 0) >> np.uint64(11)).astype(np.float64) * (1.0 / (1 << 53))
            r0 = _uniform(seed, n, 2, 4)
            nr = 1 + _uniform(seed, n, 3, 4)
            return {
                "n": n, "kind": np.minimum(np.searchsorted(cdf, u), self.n_kinds - 1), "pid": _uniform(seed, n, 1, 4096),
                "r0": r0, "nr": nr,     # roles: role_names[(r0 + q) % 4] for q < nr
                "scope": np.where(_prob(seed, n, 5, 0.05), 5, _uniform(seed, n, 4, 5)),
                "tier": _uniform(seed, n, 6, 3), "jtier": _uniform(seed, n, 7, 4), "level": _uniform(seed, n, 8, 10),
                "min_level": _uniform(seed, n, 9, 10), "nreg": 1 + _uniform(seed, n, 10, 3), "reg0": _uniform(seed, n, 11, 4),
                "mreg": _uniform(seed, n, 12, 4), "own": _prob(seed, n, 13, 0.3), "public": _prob(seed, n, 14, 0.5),
                "tagsel": _uniform(seed, n, 15, 4), "grant": _uniform(seed, n, 16, 4), "aud": 1 + _uniform(seed, n, 17, 3),
                "svc": _prob(seed, n, 18, 0.5), "deploy": _prob(seed, n, 19, 0.5), "expired": _prob(seed, n, 20, 0.3),
                "iss": _prob(seed, n, 21, 0.7),
            }
        finally:
            _TLS.start = 0

    def inputs(self, f, idx):
        out = []
        heat = ["hot", "warm", "cold", "frozen"]
        for i in idx:
            pid = f"p{f['pid'][i]}"
            kind = f"kind_{f['kind'][i]}"
            tier = self.tiers[f["tier"][i]]
            gk = [kind, f"kind_{(f['kind'][i] + 1) % self.n_kinds}", "other", "misc"][f["grant"][i]]
            meta = {"tags": {t: heat[(f["tagsel"][i] + q) % 4] for q, t in enumerate(self.tiers[: 1 + f["tagsel"][i] % 3])},
                    "region": self.regions[f["mreg"][i]]}
            if f["tagsel"][i] != 3:
                meta["owner"] = pid if f["own"][i] else "p-someone"
            aud = (["svc"] if f["svc"][i] else []) + [f"aud{q}" for q in range(f["aud"][i])]
            jwt = {"iss": "https://issuer.example" if f["iss"][i] else "https://other.example", "aud": aud, "sub": pid,
                   "scope": " ".join((["deploy"] if f["deploy"][i] else []) + ["read", "list"]),
                   "tier": (self.tiers + ["banned"])[f["jtier"][i]],
                   "exp_ts": "2020-01-01T00:00:00Z" if f["expired"][i] else "2031-06-01T12:00:00Z"}
            req = {"requestId": str(i), "actions": list(self.actions),
                   "principal": {"id": pid, "roles": [self.role_names[(int(f["r0"][i]) + q) % 4] for q in range(int(f["nr"][i]))],
                                 "attr": {"tier": tier, "level": int(f["level"][i]),
                                          "regions": [self.regions[(f["reg0"][i] + q) % 4] for q in range(f["nreg"][i])],
                                          "grants": {gk: ["read", "write"] if f["grant"][i] % 2 == 0 else ["read"], "zzz": ["write"]}}},
                   "resource": {"kind": kind, "id": f"r{i}", "attr": {"meta": meta, "public": bool(f["public"][i]), "min_level": int(f["min_level"][i])}},
                   "auxData": {"jwt": jwt}}
            sc = self.req_scopes[f["scope"][i]]
            if sc:
                req["resource"]["scope"] = sc
            out.append(req)
        return out

    def columns(self, f, enc: Encoder) -> Batch:
        """Vectorised column builder (numpy): what the generic encoder makes of inputs(f, ...), without the per-request Python.
        Every request gets its own heap records (its lists, its two maps and the nested lists), as an encoder would write them."""
        n = f["n"]
        nts = enc.n_table_strings
        extra: list = []
        pos_of: dict = {}

        def ids_for(strings):
            out = []
            for s_ in strings:
                i_ = enc.table_strings.get(s_)
                if i_ is None:
                    bkey = s_.encode("utf-8")
                    j = pos_of.get(bkey)
                    if j is None:
                        j = len(extra)
                        pos_of[bkey] = j
                        extra.append(bkey)
                    i_ = nts + j
                out.append(int(i_))
            return np.array(out, dtype=np.uint64)

        heat = ["hot", "warm", "cold", "frozen"]
        pid_ids = ids_for([f"p{i}" for i in range(4096)])
        someone = ids_for(["p-someone"])[0]
        kind_ids = ids_for([f"kind_{k}" for k in range(self.n_kinds)])
        other_misc = ids_for(["other", "misc"])
        zzz, read, write, svc = (ids_for([x])[0] for x in ("zzz", "read", "write", "svc"))
        tier_ids, heat_ids, region_ids = ids_for(self.tiers), ids_for(heat), ids_for(self.regions)
        jtier_ids = ids_for(self.tiers + ["banned"])
        aud_ids = ids_for([f"aud{q}" for q in range(3)])
        iss_ids = ids_for(["https://other.example", "https://issuer.example"])
        scope_ids = ids_for(["read list", "deploy read list"])
        exp_ids = ids_for(["2031-06-01T12:00:00Z", "2020-01-01T00:00:00Z"])

        kvals, class_list = _kind_classes(enc, [f"kind_{k}" for k in range(self.n_kinds)])
        hdr0 = np.zeros((n, 4), dtype=np.uint32)
        hdr0[:, 0] = pid_ids[f["pid"]]
        hdr0[:, 1] = kvals[f["kind"]]
        sc_ids = np.array([enc.resolve_scope(s_) for s_ in self.req_scopes], dtype=np.uint32)
        hdr0[:, 2] = sc_ids[f["scope"]]
        hdr0[:, 3] = enc.resolve_scope("")
        hdr1 = np.zeros(n, dtype=np.dtype([("rv", "<u2"), ("pv", "<u2"), ("aset", "<u4")]))
        hdr1["rv"] = enc.version_ids.get("default", L.NONE16)
        hdr1["pv"] = hdr1["rv"]
        rmap = np.array([enc.role_ids.get(r, L.ROLE_UNKNOWN) for r in self.role_names], dtype=np.uint32)
        roles = np.stack([np.where(q < f["nr"], rmap[(f["r0"] + q) % 4], np.uint32(L.ROLE_PAD)) for q in range(4)]).astype(np.uint32)

        box_s = lambda ids: _box(L.V64_STRING, ids)   # noqa: E731
        batch_bit = np.uint64(L.V64_HEAP_BATCH_BIT)
        svc_i = f["svc"].astype(np.int64)
        # principal.attr.regions; jwt.aud = (["svc"]) + aud0 ..
        reg_w, reg_off = _ragged_lists(f["nreg"], lambda req, pos: box_s(region_ids[(f["reg0"][req] + pos) % 4]))
        aud_w, aud_off = _ragged_lists(svc_i + f["aud"], lambda req, pos: box_s(np.where((svc_i[req] == 1) & (pos == 0), svc, aud_ids[np.maximum(pos - svc_i[req], 0)])))
        # resource.attr.meta.tags = {tiers[q]: heat[(tagsel + q) % 4] for q < 1 + tagsel % 3}: [m, keys.., values..]
        m = 1 + f["tagsel"] % 3
        tag_w, tag_off = _ragged_lists(2 * m, lambda req, pos: box_s(np.where(pos < m[req], tier_ids[np.minimum(pos, 2)],
                                                                                heat_ids[(f["tagsel"][req] + pos - m[req]) % 4])), head=m)
        # principal.attr.grants = {gk: ["read", "write"] | ["read"], "zzz": ["write"]}: two nested lists, then [2, gk, zzz, ref, ref]
        rw = (f["grant"] % 2 == 0)
        l1_w, l1_off = _ragged_lists(np.where(rw, 2, 1), lambda req, pos: box_s(np.where(pos == 0, read, write)))
        l2_w = np.empty((n, 2), dtype=np.uint64)
        l2_w[:, 0] = 1
        l2_w[:, 1] = box_s(np.full(n, write, dtype=np.uint64))
        gk = np.where(f["grant"] == 0, kind_ids[f["kind"]], np.where(f["grant"] == 1, kind_ids[(f["kind"] + 1) % self.n_kinds], other_misc[np.maximum(f["grant"] - 2, 0)]))
        base_reg, base_aud = 0, len(reg_w)
        base_tag = base_aud + len(aud_w)
        base_l1 = base_tag + len(tag_w)
        base_l2 = base_l1 + len(l1_w)
        base_map = base_l2 + 2 * n
        gm = np.empty((n, 5), dtype=np.uint64)
        gm[:, 0] = 2
        gm[:, 1] = box_s(gk)
        gm[:, 2] = box_s(np.full(n, zzz, dtype=np.uint64))
        gm[:, 3] = _box(L.V64_LIST, (l1_off + base_l1).astype(np.uint64) | batch_bit)
        gm[:, 4] = _box(L.V64_LIST, (np.arange(n, dtype=np.int64) * 2 + base_l2).astype(np.uint64) | batch_bit)
        heap = np.concatenate([reg_w, aud_w, tag_w, l1_w, l2_w.reshape(-1), gm.reshape(-1)])
        absent = np.uint64((L.V64_BOX_BASE | L.V64_ABSENT) << 48)
        vals = {
            ("aux_data", "jwt", "scope"): box_s(scope_ids[f["deploy"].astype(np.int64)]),
            ("aux_data", "jwt", "exp_ts"): box_s(exp_ids[f["expired"].astype(np.int64)]),
            ("aux_data", "jwt", "iss"): box_s(iss_ids[f["iss"].astype(np.int64)]),
            ("aux_data", "jwt", "aud"): _box(L.V64_LIST, (aud_off + base_aud).astype(np.uint64) | batch_bit),
            ("aux_data", "jwt", "tier"): box_s(jtier_ids[f["jtier"]]),
            ("principal", "attr", "level"): f["level"].astype(np.float64).view(np.uint64),
            ("principal", "attr", "tier"): box_s(tier_ids[f["tier"]]),
            ("principal", "attr", "regions"): _box(L.V64_LIST, (reg_off + base_reg).astype(np.uint64) | batch_bit),
            ("principal", "attr", "grants"): _box(L.V64_MAP, (np.arange(n, dtype=np.int64) * 5 + base_map).astype(np.uint64) | batch_bit),
            ("resource", "kind"): box_s(kind_ids[f["kind"]]),
            ("resource", "attr", "public"): _box(L.V64_BOOL, f["public"].astype(np.uint64)),
            ("resource", "attr", "min_level"): f["min_level"].astype(np.float64).view(np.uint64),
            ("resource", "attr", "meta", "owner"): np.where(f["tagsel"] == 3, absent, box_s(np.where(f["own"], pid_ids[f["pid"]], someone))),
            ("resource", "attr", "meta", "tags"): _box(L.V64_MAP, (tag_off + base_tag).astype(np.uint64) | batch_bit),
            ("resource", "attr", "meta", "region"): box_s(region_ids[f["mreg"]]),
        }
        slots = np.zeros((max(len(enc.slots), 1), n), dtype=np.uint64)
        for s_, path in enumerate(enc.slots):
            slots[s_] = vals[path]
        return _finish_batch(enc, n, hdr0, hdr1, roles, slots, heap, extra, class_list, [tuple(self.actions)], 8)

    def bytes_per_request(self):
        return 489   # SURVEY.md 8(d): 24 + 4*4 + 8*24 + 256 + 1


WORKLOADS = {"C1": C1, "C2": C2, "C3": C3, "C5": C5}


def columns_parallel(w, n, start, enc: Encoder, chunk=1 << 20, threads=None) -> Batch:
    """w.columns(w.fields(n, start), enc) built chunk by chunk on a thread pool (numpy releases the GIL) and merged: the
    per-request columns are concatenated, list / map references into the batch heap are rebased.  For workloads whose
    batch-level tables (string dictionary, kind classes, action sets) do not depend on the requests (C2, C3)."""
    from concurrent.futures import ThreadPoolExecutor
    import os
    if n <= chunk:
        return w.columns(w.fields(n, start=start), enc)
    threads = threads or min(32, os.cpu_count() or 1)
    spans = [(s0, min(chunk, n - s0)) for s0 in range(0, n, chunk)]
    with ThreadPoolExecutor(max_workers=threads) as ex:
        parts = list(ex.map(lambda sp: w.columns(w.fields(sp[1], start=start + sp[0]), enc), spans))
    first = parts[0]
    for p in parts[1:]:
        for ci in (5, 6, 7, 8, 9, 10, 11):
            assert np.array_equal(np.asarray(p.columns[ci]), np.asarray(first.columns[ci])), "batch-level tables differ between chunks"
    batch_bit = np.uint64(L.V64_HEAP_BATCH_BIT)
    lo48 = np.uint64((1 << 48) - 1)

    def rebase(a, base):
        """heap references (LIST / MAP boxes with the batch bit) inside `a` move by `base` words"""
        if base == 0:
            return a
        tag = (a >> np.uint64(48)).astype(np.uint32)
        ref = ((tag == (L.V64_BOX_BASE | L.V64_LIST)) | (tag == (L.V64_BOX_BASE | L.V64_MAP))) & ((a & batch_bit) != 0)
        out = a.copy()
        out[ref] = (a[ref] & ~lo48) | ((a[ref] & lo48) + np.uint64(base))
        return out

    bases = np.cumsum([0] + [len(p.columns[4]) for p in parts[:-1]])
    hdr0 = np.concatenate([p.columns[0] for p in parts], axis=0)
    hdr1 = np.concatenate([p.columns[1] for p in parts], axis=0)
    roles = np.concatenate([p.columns[2] for p in parts], axis=1)
    slots = np.concatenate([rebase(p.columns[3], int(b)) for p, b in zip(parts, bases)], axis=1)
    heap = np.concatenate([rebase(np.asarray(p.columns[4]), int(b)) for p, b in zip(parts, bases)])
    cols = [hdr0, hdr1, roles, slots, heap] + list(first.columns[5:])
    return Batch(n, first.max_actions, first.role_cols, cols, None, first.n_pass, first.kc)


def build(workload, globals_=None):
    """-> (rule table, FlatTable, Encoder)"""
    from cerbos_b200.policy.compile import build_rule_table
    from cerbos_b200.table.flatten import flatten
    rt = build_rule_table(workload.policies())
    ft = flatten(rt, globals_=globals_)
    return rt, ft, Encoder(ft.manifest)
