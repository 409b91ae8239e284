"""`Engine.Check` over the GPU evaluator -- host-side mirror of the reference's Go entry point.

Mirrors ``(*Engine).Check(ctx, []*enginev1.CheckInput, ...CheckOpt) ([]*enginev1.CheckOutput, error)``
(internal/engine/engine.go:222-246) and the ``evaluator.Conf`` / ``CheckOpt`` knobs that shape a decision
(internal/evaluator/conf.go:29-52, evaluator.go:21-64): Globals, DefaultPolicyVersion, DefaultScope,
LenientScopeSearch, NowFunc.  Inputs and outputs use protojson-shaped dicts (the same shape as the
reference's engine golden files).  Conventions kept: outputs are index-aligned with inputs; every action of
an input appears in its output with EFFECT_ALLOW or EFFECT_DENY; any failure raises (fails the whole call);
``now`` is fixed once per call.

``check(..., include_meta=True)`` also fills ``policy`` / ``scope`` of every action and ``effectiveDerivedRoles`` (the
reference's IncludeMeta responses, cerbos_svc.go:291-311) from the device's metadata plane (cgpu_check_meta).
``check(..., include_outputs=True)`` also fills ``outputs`` of every input: the rule outputs (ruletable.go:1065-1106) in the
reference's emission order, from the device (cgpu_check_outputs), with the metadata of include_meta.  ``has_outputs`` tells
whether the table declares any; ``unlowered_outputs`` lists those the device cannot evaluate (a request reaching one fails).
Not produced (SURVEY.md 8(f)): validation errors, audit trail.
"""
from __future__ import annotations

import time

from . import capi
from .encode import Encoder
from .policy.compile import build_rule_table
from .table import layout as L
from .table.flatten import flatten

EFFECT_NAMES = {1: "EFFECT_ALLOW", 2: "EFFECT_DENY"}


class Engine:
    def __init__(self, policies, globals_=None, default_policy_version="default", default_scope="",
                 lenient_scope_search=False, device: int = 0):
        self.conf = dict(globals_=globals_ or {}, default_policy_version=default_policy_version,
                         default_scope=default_scope, lenient_scope_search=lenient_scope_search)
        self.ctx = capi.Context(device)
        self.table = None
        self.encoder = None
        self.reload(policies)

    @classmethod
    def from_rule_table_bundle(cls, bundle: bytes, key=None, **conf):
        """An engine over a serialized runtimev1.RuleTable (rule-table bundle, storage/hub/ruletable_bundle.go:36-87).
        key: the bundle's encryption key (32 bytes or 64 hex digits) for an encrypted bundle (`*.crrts`), None for a plain one."""
        from .table.ruletable_pb import decode_rule_table
        if key is not None:
            from .table.bundle_crypto import decrypt_stream
            bundle = decrypt_stream(key, bundle)
        self = cls.__new__(cls)
        self.conf = dict(globals_=conf.get("globals_") or {}, default_policy_version=conf.get("default_policy_version", "default"),
                         default_scope=conf.get("default_scope", ""), lenient_scope_search=conf.get("lenient_scope_search", False))
        self.ctx = capi.Context(conf.get("device", 0))
        self.table = None
        self.encoder = None
        self._install(decode_rule_table(bundle))
        return self

    def reload(self, policies):
        """Build-then-swap, like Manager.reload (internal/ruletable/manager.go:88-124): on failure the
        previous table stays in place."""
        self._install(build_rule_table(policies))

    def _install(self, rt):
        ft = flatten(rt, globals_=self.conf["globals_"])
        new_table = self.ctx.load_table(ft.blob)
        old, self.table = self.table, new_table
        self.flat = ft
        self.encoder = Encoder(ft.manifest, default_version=self.conf["default_policy_version"],
                               default_scope=self.conf["default_scope"],
                               lenient_scope_search=self.conf["lenient_scope_search"])
        if old is not None:
            old.release()

    @property
    def has_outputs(self) -> bool:
        return bool(self.flat.manifest.get("output_sources"))

    @property
    def unlowered_outputs(self) -> list:
        """[{"policy", "rule", "kind", "when", "reason"}]: outputs without a device program."""
        return list(self.flat.manifest.get("unlowered_outputs") or [])

    def check_effects(self, inputs, now_ns=None):
        """-> (Batch, uint8[n, K] effects)"""
        if now_ns is None:
            now_ns = time.time_ns()
        batch = self.encoder.encode(inputs)
        flags = L.BATCH_FLAG_LENIENT if self.conf["lenient_scope_search"] else 0
        eff = self.table.check(batch.columns, batch.n, batch.max_actions, now_ns, flags)
        return batch, eff

    def check(self, inputs, now_ns=None, include_meta=False, include_outputs=False):
        """-> list of CheckOutput dicts, index-aligned with `inputs`.  include_meta: also `policy` / `scope` per action
        and `effectiveDerivedRoles` (ruletable.go:753-782), through the metadata plane of the device.  include_outputs:
        that, and `outputs` ([{"src", "action", "val"}] in emission order)."""
        if not inputs:
            return []
        if include_meta or include_outputs:
            return self._check_with_meta(inputs, now_ns, include_outputs)
        batch, eff = self.check_effects(inputs, now_ns)
        outs = []
        for i, inp in enumerate(inputs):
            actions = {}
            for k, a in enumerate(inp.get("actions") or []):
                actions[a] = {"effect": EFFECT_NAMES[int(eff[i, k])]}
            outs.append({"requestId": inp.get("requestId", ""), "resourceId": (inp.get("resource") or {}).get("id", ""),
                         "actions": actions})
        return outs

    OUTPUT_STRIDE = 4096   # first guess of an output record's size; a call whose records need more is repeated once with that

    def _check_with_meta(self, inputs, now_ns=None, include_outputs=False):
        from . import meta as M
        if now_ns is None:
            now_ns = time.time_ns()
        batch = self.encoder.encode(inputs)
        flags = L.BATCH_FLAG_LENIENT if self.conf["lenient_scope_search"] else 0
        man = self.flat.manifest
        entries = None
        if include_outputs:
            from . import outputs as O
            stride = self.OUTPUT_STRIDE
            try:
                eff, am, rm, rec, _ = self.table.check_outputs(batch.columns, batch.n, batch.max_actions, stride, now_ns, flags)
            except capi.CgpuError as e:
                if not getattr(e, "bytes_needed", 0):
                    raise
                stride = (e.bytes_needed + 7) // 8 * 8
                eff, am, rm, rec, _ = self.table.check_outputs(batch.columns, batch.n, batch.max_actions, stride, now_ns, flags)
            entries = O.decode(rec, stride, man, [inp.get("actions") or [] for inp in inputs])
        else:
            eff, am, rm = self.table.check_meta(batch.columns, batch.n, batch.max_actions, now_ns, flags)
        outs = []
        for i, inp in enumerate(inputs):
            p, r = inp.get("principal") or {}, inp.get("resource") or {}
            p_ver = p.get("policyVersion") or self.conf["default_policy_version"]
            r_ver = r.get("policyVersion") or self.conf["default_policy_version"]
            actions = {}
            for k, a in enumerate(inp.get("actions") or []):
                policy, scope = M.decode_action(int(am[i, k]), rm[i], man, p.get("id", ""), r.get("kind", ""), p_ver, r_ver)
                actions[a] = {"effect": EFFECT_NAMES[int(eff[i, k])], "policy": policy, "scope": scope}
            outs.append({"requestId": inp.get("requestId", ""), "resourceId": r.get("id", ""), "actions": actions,
                         "effectiveDerivedRoles": M.decode_edr(int(rm[i]["effective_derived_roles"]), man)})
            if entries is not None:
                outs[-1]["outputs"] = entries[i]
        return outs

    def close(self):
        if self.table is not None:
            self.table.release()
            self.table = None
        self.ctx.close()
