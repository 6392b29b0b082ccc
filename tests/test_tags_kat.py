"""CPU: known answers of particle tags (DESIGN.md §8, "Particle tags"): the census quantisation restated with NumPy, the version-4 state file
written from its documented layout and read by blub_state_info, and the scene key "tag" as blub_scene_info parses it.  No GPU needed."""
import json
import os
import struct
import zlib
from fractions import Fraction

import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from tests import test_flow_kat as FK, test_state_file as SF, util

BLUB_ERR_PARSE = 5
FRAC = F.TAG_CENSUS_FRAC_BITS


def census_fixed(x):
    """What one particle adds to a census sum: rint(float64(x) * 2^16) as int64 (round half to even)."""
    return np.rint(np.asarray(x, dtype=np.float32).astype(np.float64) * (1 << FRAC)).astype(np.int64)


# ---- census quantisation ------------------------------------------------------------------------------------------------
EDGES = [0.0, -0.0, 1.0, -1.0, 0.5 / 65536, 1.5 / 65536, 2.5 / 65536, -0.5 / 65536, -1.5 / 65536, -2.5 / 65536, 3.5 / 65536,
         1.0001, 1.001001, 1023.99994, 1.0 - 2.0 ** -24, 2.0 ** -17, 3 * 2.0 ** -18, 2.0 ** -149, -(2.0 ** -149), 2.0 ** -126,
         float(np.float32(-1.2345678)), 2.0 ** 20, -(2.0 ** 20), 2.0 ** 20 - 2.0 ** -4, 1.00000012]


def test_the_float64_restatement_rounds_the_exact_product_to_nearest_even():
    x = np.asarray(EDGES, dtype=np.float32)
    got = census_fixed(x)
    want = [round(Fraction(float(v)) * (1 << FRAC)) for v in x]  # Python rounds a Fraction half to even
    assert got.tolist() == want
    # the float32 product the kernel rounds is exact: the same number as the float64 product
    assert np.array_equal((x * np.float32(65536)).astype(np.float64), x.astype(np.float64) * 65536)
    assert np.array_equal(np.rint(x * np.float32(65536)).astype(np.int64), got)
    # halves go to the even neighbour, signs are symmetric
    assert census_fixed([0.5 / 65536, 1.5 / 65536, 2.5 / 65536]).tolist() == [0, 2, 2]
    assert census_fixed([-0.5 / 65536, -1.5 / 65536, -2.5 / 65536]).tolist() == [0, -2, -2]


def test_random_values_in_the_documented_ranges_agree_with_exact_rounding():
    rng = np.random.default_rng(3)
    pos = rng.uniform(0, 1024, 2000).astype(np.float32)
    vel = (rng.standard_normal(2000) * rng.choice([1e-6, 1e-2, 1.0, 1e3, 1e6], 2000)).astype(np.float32)
    for x in (pos, vel):
        assert census_fixed(x).tolist() == [round(Fraction(float(v)) * 65536) for v in x]


def test_sums_stay_exact_at_the_documented_limits():
    # 2^26 particles per tag at a position below 2^10 and at |v| = 2^20: the sums fit int64 with room to spare
    assert (2 ** 26) * int(census_fixed(np.float32(1024 - 2 ** -14))) < 2 ** 63
    assert (2 ** 26) * int(census_fixed(np.float32(2 ** 20))) < 2 ** 63
    # and every position contribution is an integer of at most 26 bits, exactly representable in the float64 centroid
    assert int(census_fixed(np.float32(1024 - 2 ** -14))) < 2 ** 26


# ---- state file, format version 4 -------------------------------------------------------------------------------------
SOURCE_TAGS = [0xFFFFFFFF] + [0] * 15


def tags_payload(tags=SOURCE_TAGS):
    return struct.pack("<16I", *tags)


def state_v4(payload14=None, version=4):
    """The version-2 layout of DESIGN.md §8 with format_version = 4 and section 14 followed by u32 source_tags[16] (1056 bytes)."""
    h = bytearray(SF.header(version=version))
    struct.pack_into("<I", h, SF.HEADER_BYTES - 8, 14)  # num_sections
    struct.pack_into("<I", h, SF.HEADER_BYTES - 4, zlib.crc32(bytes(h[:SF.HEADER_BYTES - 4])))
    out = bytes(h)
    for sid, p in enumerate(SF.payloads(), start=1):
        out += SF.section(sid, p)
    return out + SF.section(14, FK.flow_payload() + tags_payload() if payload14 is None else payload14)


def test_a_version_4_file_from_the_documented_layout_is_accepted(tmp_path):
    assert len(FK.flow_payload() + tags_payload()) == 1056
    info = blub_b200.state_info(SF.write(tmp_path, state_v4()))
    assert (info.num_particles, info.step_count, info.format_version) == (SF.NUM_PARTICLES, SF.STEP_COUNT, 4)


def _bad_crc():
    b = bytearray(state_v4())
    b[-8] ^= 0x01  # a byte of the source tags
    return bytes(b)


@pytest.mark.parametrize("case,make,needle", [
    ("truncated", lambda: state_v4()[:-4], "bytes"),
    ("one byte too many", lambda: state_v4() + b"\0", "bytes"),
    ("bad checksum of section 14", _bad_crc, "checksum"),
    ("version 4 with a version-2-sized section 14", lambda: state_v4(FK.flow_payload()), "bytes"),
    ("version 2 with a version-4-sized section 14", lambda: state_v4(version=2), "bytes"),
])
def test_malformed_version_4_files_are_parse_errors(tmp_path, case, make, needle):
    rc, msg, _ = SF.info_rc(SF.write(tmp_path, make()))
    assert rc == BLUB_ERR_PARSE and needle in msg, (case, rc, msg)


@pytest.mark.parametrize("version", [0, 3, 5])
def test_versions_other_than_1_2_and_4_are_parse_errors(tmp_path, version):
    """Version 3 is not a format: a file that claims it is refused even with the layout of version 4."""
    rc, msg, _ = SF.info_rc(SF.write(tmp_path, state_v4(version=version)))
    assert rc == BLUB_ERR_PARSE and f"version {version} is not supported" in msg, msg


# ---- scene key "tag" --------------------------------------------------------------------------------------------------
def test_the_tagged_scene_and_the_largest_tag_are_accepted(tmp_path):
    info = blub_b200.scene_info(util.scene_path("tap_tagged_small"))
    assert tuple(info.grid_dimension) == (32, 32, 32) and info.num_fluid_cubes == 2
    sc = json.load(open(util.scene_path("dam_small")))
    sc["fluid"]["fluid_cubes"][0]["tag"] = 4294967295
    path = tmp_path / "max.json"
    path.write_text(json.dumps(sc))
    assert blub_b200.scene_info(str(path)).num_fluid_cubes == 1


@pytest.mark.parametrize("where", ["fluid_cubes", "sources"])
@pytest.mark.parametrize("value", [-1, 1.5, 4294967296, 1e20, "7", None, True, [3]])
def test_bad_tag_values_are_parse_errors(tmp_path, where, value):
    sc = json.load(open(util.scene_path("tap_tagged_small")))
    sc["fluid"][where][0]["tag"] = value
    path = tmp_path / "bad.json"
    path.write_text(json.dumps(sc))
    out = F.SceneInfo()
    assert F.lib().blub_scene_info(os.fsencode(str(path)), out) == BLUB_ERR_PARSE
    assert b"tag" in F.lib().blub_last_error()
