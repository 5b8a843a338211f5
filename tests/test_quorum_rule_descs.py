"""Group descriptors carry the quorum rule and the proposer where the C struct ibft_group_desc keeps them (no GPU needed)."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import ibft_b200 as ib
from conftest import ROOT


def header_defines():
    src = open(os.path.join(ROOT, "include", "ibft_verify.h")).read()
    return {k: int(v, 0) for k, v in re.findall(r"#define (IBFT_(?:QUORUM|PROPOSER)_\w+) (0x[0-9A-Fa-f]+|\d+)u", src)}


def test_constants_match_the_header():
    d = header_defines()
    assert (d["IBFT_QUORUM_DEFAULT"], d["IBFT_QUORUM_PREPREPARE"], d["IBFT_QUORUM_PREPARE"]) == (
        ib.QUORUM_DEFAULT, ib.QUORUM_PREPREPARE, ib.QUORUM_PREPARE)
    assert (d["IBFT_PROPOSER_NONE"], d["IBFT_PROPOSER_UNSET"]) == (ib.PROPOSER_NONE, ib.PROPOSER_UNSET)
    assert d["IBFT_QUORUM_RULE_MASK"] == 3


def test_default_descriptors_are_zero_in_flags_and_reserved():
    g = ib.group_descs(5, slot=[0, 1, 2, ib.NO_TABLE, 3], slot_height={0: 10, 1: 11, 2: 12, 3: 13})
    assert [int(x) for x in g["flags"]] == [0] * 5 and [int(x) for x in g["reserved"]] == [0] * 5
    assert [int(x) for x in g["height"]] == [10, 11, 12, 0, 13]
    # a proposer given for groups whose rule has none is not stored
    g = ib.group_descs(3, rule=[ib.QUORUM_DEFAULT, ib.QUORUM_PREPREPARE, ib.QUORUM_DEFAULT], proposer=7)
    assert [int(x) for x in g["reserved"]] == [0, 0, 0]


def test_rule_and_proposer_land_at_the_struct_offsets():
    """The packed bytes: flags (rule in bits 0-1) at byte 2 as u16 LE, the proposer at byte 4 as u32 LE, per GROUP_DTYPE."""
    rules = [ib.QUORUM_PREPARE, ib.QUORUM_PREPREPARE, ib.QUORUM_PREPARE, ib.QUORUM_PREPARE, ib.QUORUM_DEFAULT]
    props = [0x01020304, 9, ib.PROPOSER_NONE, ib.PROPOSER_UNSET, 5]
    g = ib.group_descs(5, slot=7, rule=rules, proposer=props, slot_height={7: 0x1122334455667788})
    raw = g.tobytes()
    f_off, r_off, h_off = (ib.GROUP_DTYPE.fields[k][1] for k in ("flags", "reserved", "height"))
    assert (ib.GROUP_DTYPE.fields["table_slot"][1], f_off, r_off, h_off) == (0, 2, 4, 8)
    for i in range(5):
        rec = raw[16 * i: 16 * (i + 1)]
        assert int.from_bytes(rec[0:2], "little") == 7
        assert int.from_bytes(rec[f_off:f_off + 2], "little") & 3 == rules[i]
        assert int.from_bytes(rec[r_off:r_off + 4], "little") == (props[i] if rules[i] == ib.QUORUM_PREPARE else 0)
        assert int.from_bytes(rec[h_off:h_off + 8], "little") == 0x1122334455667788
    with pytest.raises(ValueError):
        ib.group_descs(3, rule=[ib.QUORUM_PREPARE] * 2)


@pytest.mark.skipif(shutil.which("cc") is None, reason="no C compiler")
def test_group_dtype_offsets_equal_the_c_struct(tmp_path):
    """offsetof() of ibft_group_desc as a C compiler lays it out equals GROUP_DTYPE's offsets."""
    src = tmp_path / "off.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ibft_verify.h"\n'
                   "int main(void) { printf(\"%zu %zu %zu %zu %zu\\n\", offsetof(ibft_group_desc, table_slot), "
                   "offsetof(ibft_group_desc, flags), offsetof(ibft_group_desc, reserved), offsetof(ibft_group_desc, height), "
                   "sizeof(ibft_group_desc)); return 0; }\n")
    exe = tmp_path / "off"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [ib.GROUP_DTYPE.fields[k][1] for k in ("table_slot", "flags", "reserved", "height")] + [ib.GROUP_DTYPE.itemsize]
    assert np.dtype(ib.GROUP_DTYPE).itemsize == 16
