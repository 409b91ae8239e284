"""Pins the CPU oracle against the reference's own golden vectors (SURVEY.md §8c).

Fixtures under tests/golden/ are extracted from the cerbos/cerbos test data by
tests/golden/make_golden.py.
"""
import pytest

from cerbos_b200.cel.parser import parse
from helpers import EFFECT_NAMES, engine_decisions, load_golden, store_rule_table
from oracle.activation import build_activation, build_request
from oracle.celeval import CelError, eval_expr, parse_timestamp
from oracle.check import CheckOracle

# internal/engine/evaluator_test.go:27-30
CEL_EVAL_NOW = parse_timestamp("2021-04-22T10:05:20.021-05:00")


def _sat(cond, act, now):
    if "expr" in cond:
        try:
            return eval_expr(parse(cond["expr"]), act, now) is True
        except CelError:
            return False
    if "all" in cond:
        return all(_sat(c, act, now) for c in cond["all"]["of"])
    if "any" in cond:
        return any(_sat(c, act, now) for c in cond["any"]["of"])
    return not any(_sat(c, act, now) for c in cond["none"]["of"])


@pytest.mark.parametrize("tc", load_golden("cel_eval.json"), ids=lambda tc: tc["file"])
def test_cel_eval_goldens(tc):
    act = build_activation(build_request(tc["request"]))
    assert _sat(tc["condition"], act, CEL_EVAL_NOW) == tc["want"]


_LIB = [tc for tc in load_golden("cerbos_lib_test.json")]


@pytest.mark.parametrize("tc", _LIB, ids=lambda tc: tc["expr"][:60])
def test_cerbos_lib_table(tc):
    """internal/conditions/cerbos_lib_test.go:26-134 -- every expression is true (or errors).
    The reference runs it with the real wall clock, so `now` only has to be later than 2021-05-01."""
    now = parse_timestamp("2026-01-01T00:00:00Z")
    act = build_activation(build_request({}))
    try:
        v = eval_expr(parse(tc["expr"]), act, now)
        err = False
    except CelError:
        err = True
    assert err == tc["wantErr"]
    if not err:
        assert v is True


def test_engine_goldens_effect_policy_scope():
    """166 decisions of internal/test/testdata/engine*, runner internal/engine/engine_test.go:50-234."""
    orc = CheckOracle(store_rule_table(), globals_={"environment": "test"})
    now = parse_timestamp("2024-01-01T00:00:00Z")
    n = n_out = 0
    for cid, lenient, inp, want in engine_decisions():
        got = orc.check(inp, now, lenient=lenient)
        for action, w in want["actions"].items():
            g = got["actions"][action]
            assert EFFECT_NAMES[g["effect"]] == w["effect"], (cid, action)
            assert g["policy"] == w.get("policy", ""), (cid, action)
            assert g["scope"] == w.get("scope", ""), (cid, action)
            n += 1
        wedr = want.get("effectiveDerivedRoles", want.get("effective_derived_roles")) or []
        assert sorted(wedr) == got["effectiveDerivedRoles"], cid
        # rule outputs (ruletable.go:1065-1106): the engine test compares them as a set (engine_test.go sorts by src / action)
        key = lambda o: (o["src"], o["action"], repr(o["val"]))  # noqa: E731
        assert sorted(got["outputs"], key=key) == sorted(want.get("outputs") or [], key=key), cid
        n_out += len(want.get("outputs") or [])
    assert n == 166 and n_out == 6


def test_rule_outputs_of_the_api_goldens():
    """Rule outputs recorded by the API-level CheckResources goldens (cr_case_0*.yaml: nested maps and lists, values built
    from the principal, a principal-policy rule's output): oracle #1, ruletable.go:1065-1106 + :1443-1465."""
    from helpers import check_resources_api_outputs
    orc = CheckOracle(store_rule_table(), globals_={"environment": "test"})
    key = lambda o: (o["src"], o["action"])  # noqa: E731
    n = 0
    for f, ci, want in check_resources_api_outputs():
        got = orc.check(ci)["outputs"]
        assert sorted(got, key=key) == sorted(want, key=key), f
        n += len(want)
    assert n == 5


def test_parent_role_index_known_answers():
    """internal/ruletable/index/index_test.go:15-60 (TestParentRoleIndex): the transitive closure of parent roles per scope.
    The hot path always asks for ONE scope (ruletable.go:865, 924: AddParentRoles(ctx, []string{resourceScope}, ...)); the
    reference's multi-scope case is the union of the per-scope answers."""
    from cerbos_b200.policy.model import RuleTable
    rt = RuleTable(rows=[], scope_parent_roles={"acme": {"manager": ["employee"], "employee": ["user"]}, "acme.hr": {"manager": ["contractor"]}})
    orc = CheckOracle(rt)
    assert sorted(orc.add_parent_roles("acme", ["manager"])) == sorted(["manager", "employee", "user"])
    assert sorted(orc.add_parent_roles("acme.hr", ["manager"])) == sorted(["manager", "contractor"])
    union = set(orc.add_parent_roles("acme", ["manager"])) | set(orc.add_parent_roles("acme.hr", ["manager"]))
    assert union == {"manager", "employee", "user", "contractor"}
    assert orc.add_parent_roles("elsewhere", ["manager"]) == ["manager"]          # (an index without the scope: the roles as given)
