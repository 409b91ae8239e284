"""The host build sets a table and a batch up through the library's own checks (cerbos_b200/csrc/cb_host.h): it refuses the
blobs and batches the library refuses, and it takes the unique-condition body only where the library may."""
import functools
import random
import struct

import numpy as np
import pytest

from hostsim import driver as hostsim
from test_uc_shapes import Case, _roles_inputs, _roles_table

HEADER = struct.Struct("<IIIIQQ")    # cb_blob_header: magic, version, n_sections, flags, total_bytes, reserved
SECTION = struct.Struct("<IIQQ")     # cb_section_desc: id, elem_bytes, offset, n_bytes
SEC_DR_NAME_STR = 30
COL_ROLES, COL_ROW_AM = 2, 11


@functools.lru_cache(maxsize=None)
def _small():
    r = random.Random(31)
    roles, kinds, docs = _roles_table(3, 2, 6, r, 0)
    return Case("small", docs, _roles_inputs(r, roles, kinds, 2, 4, 97))


def _sections(blob):
    n = HEADER.unpack_from(blob, 0)[2]
    return [(HEADER.size + i * SECTION.size, SECTION.unpack_from(blob, HEADER.size + i * SECTION.size)) for i in range(n)]


def _refused(blob, columns, c):
    with pytest.raises(RuntimeError, match=r"failed: -1$"):
        hostsim.check(blob, columns, c.b.n, c.b.max_actions, 0, c.flags, mode=1)


def test_refuses_last_section_past_the_blob_end():
    c = _small()
    blob = bytearray(c.ft.blob)
    at, (sid, eb, off, nb) = max(_sections(blob), key=lambda s: s[1][2])
    SECTION.pack_into(blob, at, sid, eb, off, len(blob) - off + 16)
    _refused(bytes(blob), c.b.columns, c)


def test_refuses_missing_required_section():
    c = _small()
    blob = bytearray(c.ft.blob)
    at, (sid, eb, off, nb) = next(s for s in _sections(blob) if s[1][0] == SEC_DR_NAME_STR)
    SECTION.pack_into(blob, at, 99, eb, off, nb)   # an id the image does not carry
    _refused(bytes(blob), c.b.columns, c)


def test_refuses_roles_column_not_a_multiple_of_requests():
    c = _small()
    cols = [np.ascontiguousarray(x) for x in c.b.columns]
    cols[COL_ROLES] = np.concatenate([cols[COL_ROLES].reshape(-1).view(np.uint8), np.zeros(4, np.uint8)])
    _refused(c.ft.blob, cols, c)


def test_refuses_undersized_row_am():
    c = _small()
    cols = [np.ascontiguousarray(x) for x in c.b.columns]
    cols[COL_ROW_AM] = cols[COL_ROW_AM].reshape(-1).view(np.uint8)[:-8]
    _refused(c.ft.blob, cols, c)


def test_role_word_without_room_for_any_role_takes_general_body():
    """Eight table roles and eight role columns fill the 64-bit role word of the lean body, leaving no room for the "any
    role" column the unique-condition body needs: modes 4 / 5 run the general body, with the decisions of oracle #2."""
    r = random.Random(32)
    roles, kinds, docs = _roles_table(8, 5, 40, r, 5)
    c = Case("nr8_rc8", docs, _roles_inputs(r, roles, kinds, 8, 4, 1001))
    assert c.nR == 8 and 5 <= c.rc <= 8 and c.nR * c.rcp == 64, (c.nR, c.rc)
    valid = c.want != 0
    for mode, body in ((0, 0), (4, 1), (5, 1)):
        got = hostsim.check(c.ft.blob, c.b.columns, c.b.n, c.b.max_actions, 0, c.flags, mode=mode)
        assert hostsim.body() == body, mode
        assert (got[valid] == c.want[valid]).all(), mode
