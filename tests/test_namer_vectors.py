"""internal/namer/namer_test.go known answers for the naming rules on the decision path: TestFQN (:17-74) and
TestFQNSpecialChars (:223-288) -- the sanitisation of resource kinds / principal ids (namer.go:213-218) that both the policy
compiler and the request encoder apply before a kind is looked up.  The Python rules (cerbos_b200/policy/namer.py) and the
native encoder's (cb_encode.h: sanitize, through a resource kind that must land in the right policy) are held to them.
Module ids (xxhash of the FQN) are not on the GPU path and not restated."""
import pytest

from cerbos_b200.policy import namer

FQN_SPECIAL = [   # (policy name, fqn function, want) -- namer_test.go:230-278
    ("resource_name", namer.resource_policy_fqn, "cerbos.resource.resource_name.vdefault/a.b.c"),
    ("my-resource@some.domain-name/path", namer.resource_policy_fqn, "cerbos.resource.my_resource_some.domain_name_path.vdefault/a.b.c"),
    ("my-resource@@@@some.domain-name//path", namer.resource_policy_fqn, "cerbos.resource.my_resource_some.domain_name_path.vdefault/a.b.c"),
    ("arn:aws:sns:us-east-1:123456789012:topic-foo", namer.resource_policy_fqn, "cerbos.resource.arn:aws:sns:us-east-1:123456789012:topic-foo.vdefault/a.b.c"),
    ("principal_name", namer.principal_policy_fqn, "cerbos.principal.principal_name.vdefault/a.b.c"),
    ("principal_name@email-domain.com", namer.principal_policy_fqn, "cerbos.principal.principal_name_email_domain.com.vdefault/a.b.c"),
    ("principal_name@@@@@email-domain.com/foo", namer.principal_policy_fqn, "cerbos.principal.principal_name_email_domain.com_foo.vdefault/a.b.c"),
    ("arn:aws:iam::123456789012:user/johndoe", namer.principal_policy_fqn, "cerbos.principal.arn:aws:iam::123456789012:user/johndoe.vdefault/a.b.c"),
]


# ids: "::" separates the parts of a pytest node id, so it is kept out of parameter ids (the IAM ARN's empty region)
@pytest.mark.parametrize("name,fn,want", FQN_SPECIAL, ids=[c[0].replace("::", ":_:") for c in FQN_SPECIAL])
def test_fqn_special_chars(name, fn, want):
    assert fn(name, "default", "a.b.c") == want


def test_fqn_forms():
    """namer_test.go:17-74 (the generated test policies: leave_request / donald_duck / my_derived_roles, version "default")"""
    assert namer.derived_roles_fqn("my_derived_roles") == "cerbos.derived_roles.my_derived_roles"
    assert namer.resource_policy_fqn("leave_request", "default", "") == "cerbos.resource.leave_request.vdefault"
    assert namer.resource_policy_fqn("leave_request", "default", "acme.base") == "cerbos.resource.leave_request.vdefault/acme.base"
    assert namer.principal_policy_fqn("donald_duck", "default", "") == "cerbos.principal.donald_duck.vdefault"
    assert namer.principal_policy_fqn("donald_duck", "default", "acme.base") == "cerbos.principal.donald_duck.vdefault/acme.base"
    assert namer.scope_parents("a.b.c") == ["a.b", "a", ""]


@pytest.mark.parametrize("kind", ["my-resource@some.domain-name/path", "my-resource@@@@some.domain-name//path", "arn:aws:sns:us-east-1:123456789012:topic-foo"])
def test_sanitised_kinds_reach_their_policy_through_both_encoders(kind):
    """A request names the resource kind as written; policy and request must meet at the sanitised name (ruletable.go:851
    namer.SanitizedResource).  Python encoder and native encoder (byte for byte) + oracle #2: ALLOW from the kind's own policy."""
    import numpy as np
    from cerbos_b200 import wire
    from cerbos_b200.encode import Encoder
    from cerbos_b200.policy.compile import build_rule_table
    from cerbos_b200.table.flatten import flatten
    from hostsim import driver as hostsim
    from oracle import cref
    pol = {"apiVersion": "api.cerbos.dev/v1", "resourcePolicy": {"resource": kind, "version": "default",
           "rules": [{"actions": ["a"], "effect": "EFFECT_ALLOW", "roles": ["user"]}]}}
    other = {"apiVersion": "api.cerbos.dev/v1", "resourcePolicy": {"resource": "something_else", "version": "default",
             "rules": [{"actions": ["a"], "effect": "EFFECT_DENY", "roles": ["user"]}]}}
    ft = flatten(build_rule_table([pol, other]))
    inp = {"principal": {"id": "p", "roles": ["user"]}, "resource": {"kind": kind, "id": "r"}, "actions": ["a"]}
    b = Encoder(ft.manifest).encode([inp])
    assert cref.check(ft.blob, b.columns, 1, 1)[0, 0] == 1
    nat = hostsim.native_encode(ft.blob, [wire.check_input(inp)])
    for a, c in zip(nat[0] if isinstance(nat, tuple) else nat, b.columns):
        assert np.asarray(a).tobytes() == np.ascontiguousarray(np.asarray(c)).tobytes()[: np.asarray(a).nbytes]
