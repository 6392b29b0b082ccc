"""CPU: the layout rule of the state file (DESIGN.md §8, "checkpoint / restart") over every combination of format version, base sections and
setting sections, as the host-only reader blub_state_info sees it.  The files are built from the known-answer helpers of each section, so the
test pins the documented format.  No GPU needed."""
import itertools
import os
import struct
import zlib

import pytest

from blub_b200 import fluid as F
from tests.test_bodies_kat import BODIES, v8_bytes
from tests.test_flow_kat import flow_payload
from tests.test_interfacial_tension_kat import it_payload
from tests.test_mesh_bodies_kat import v16_bytes
from tests.test_state_file import HEADER_BYTES, section, state_bytes
from tests.test_surface_tension_kat import st_payload
from tests.test_tag_density_kat import td_payload
from tests.test_tag_viscosity_kat import tv_payload
from tests.test_viscosity_kat import viscosity_payload

BLUB_ERR_PARSE = 5
VERSIONS = (1, 2, 3, 4, 8, 16, 32, 64, 128, 256, 512, 1024)
# the format version that introduced each optional section; section 14 written with a non-zero source tag counts as version 4
INTRO = {14: 2, 15: 8, 16: 16, 17: 32, 18: 64, 19: 128, 20: 256, 21: 512}
SETTINGS = (17, 18, 19, 20, 21)
# the base layouts: (last base section, section 14 at its 1056-byte length), bytes of sections 1 to that one
BASES = {"13": (13, False, state_bytes), "14 at 992 bytes": (14, False, lambda: state_bytes() + section(14, flow_payload())),
         "14 at 1056 bytes": (14, True, lambda: state_bytes() + section(14, flow_payload() + bytes(64))),
         "15": (15, True, lambda: v8_bytes(BODIES)), "16": (16, True, v16_bytes)}
PAYLOADS = {17: viscosity_payload(nu=3.0), 18: st_payload(), 19: td_payload(), 20: tv_payload(), 21: it_payload()}


def accepted(v, nb, tagged, extra):
    """The layout rule and the cross-section rules, restated."""
    top = max([1] + [INTRO[i] for i in list(range(14, nb + 1)) + list(extra)])
    if not (v == top or (top == 2 and v == 4)):
        return False
    if nb >= 14 and tagged != (v >= 4):
        return False
    if 20 in extra and 17 not in extra:
        return False
    if 18 in extra and 19 in extra:
        return False
    if 19 in extra and nb >= 15:
        return False
    return True


def relabel(data, version, num_sections):
    """The file with the header's format_version and num_sections rewritten and its checksum renewed."""
    out = bytearray(data)
    out[8:12] = struct.pack("<I", version)
    out[HEADER_BYTES - 8:HEADER_BYTES - 4] = struct.pack("<I", num_sections)
    out[HEADER_BYTES - 4:HEADER_BYTES] = struct.pack("<I", zlib.crc32(bytes(out[:HEADER_BYTES - 4])))
    return bytes(out)


def info_rc(path, data):
    with open(path, "wb") as f:
        f.write(data)
    L = F.lib()
    rc = L.blub_state_info(os.fsencode(path), F.StateInfo())
    return rc, L.blub_last_error().decode()


@pytest.fixture(scope="module")
def bases():
    return {name: make() for name, (_, _, make) in BASES.items()}


SUBSETS = [s for k in range(len(SETTINGS) + 1) for s in itertools.combinations(SETTINGS, k)]
ACCEPTED = {1: 1, 2: 1, 3: 0, 4: 1, 8: 1, 16: 1, 32: 4, 64: 8, 128: 4, 256: 10, 512: 30, 1024: 0}


@pytest.mark.parametrize("version", VERSIONS)
def test_the_reader_accepts_exactly_the_layouts_of_the_rule(tmp_path, bases, version):
    path = str(tmp_path / "state.blub")
    ok = []
    for name, (nb, tagged, _) in BASES.items():
        for extra in SUBSETS:
            data = relabel(bases[name], version, nb + len(extra)) + b"".join(section(i, PAYLOADS[i]) for i in extra)
            rc, msg = info_rc(path, data)
            if accepted(version, nb, tagged, extra):
                assert rc == 0, (name, extra, msg)
                ok.append((name, extra))
            else:
                assert rc == BLUB_ERR_PARSE, (name, extra, rc)
    assert len(ok) == ACCEPTED[version], ok


@pytest.mark.parametrize("version, order", [
    (64, (18, 17)), (256, (20, 17)), (256, (17, 20, 17)), (512, (17, 17, 21)), (512, (21, 21)), (512, (21, 17)), (512, (17, 21, 20)),
    (512, (18, 17, 21)), (256, (17, 19, 18, 20)), (128, (19, 17))])
def test_setting_sections_out_of_order_or_repeated_are_refused(tmp_path, bases, version, order):
    data = relabel(bases["13"], version, 13 + len(order)) + b"".join(section(i, PAYLOADS[i]) for i in order)
    rc, msg = info_rc(str(tmp_path / "state.blub"), data)
    assert rc == BLUB_ERR_PARSE, (order, msg)
