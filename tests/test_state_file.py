"""CPU: the checkpoint file format (DESIGN.md §8, "checkpoint / restart") as the host-only reader blub_state_info sees it.  The files are
written here from the documented layout with NumPy and zlib, so the test pins the format, not just the writer.  No GPU needed."""
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from tests import util

BLUB_ERR_IO, BLUB_ERR_PARSE = 4, 5
HEADER_BYTES = 144
GRID = (32, 32, 40)
MAX_PARTICLES, NUM_PARTICLES, STEP_COUNT = 1000, 300, 37
NUM_STATS = (5, 3)


def header(grid=GRID, max_num_particles=MAX_PARTICLES, num_particles=NUM_PARTICLES, version=1, magic=b"BLUBSTAT", num_stats=NUM_STATS):
    body = magic + struct.pack("<I", version) + b"blub-b200 test".ljust(32, b"\0")
    body += struct.pack("<3I", *grid) + struct.pack("<3I", max_num_particles, num_particles, STEP_COUNT)
    body += struct.pack("<2I", 8, 60)                                         # internal re-sort cadence, rebinning frequency
    body += struct.pack("<3f", 0.0, -490.5, 0.0)                              # gravity in grid units
    body += struct.pack("<fii", 0.1, 32, 4) + struct.pack("<fii", 1e-4, 128, 4)  # solver configs (velocity, density)
    body += struct.pack("<i3I", 0, 1, 1, 1)                                   # precond_mode, transfer path, solver path, graph replay
    body += struct.pack("<2I", *num_stats) + struct.pack("<I", 13)
    assert len(body) == HEADER_BYTES - 4
    return body + struct.pack("<I", zlib.crc32(body))


def section(sid, payload):
    return struct.pack("<IIQ", sid, 0, len(payload)) + payload + struct.pack("<I", zlib.crc32(payload))


def payloads():
    rng = np.random.default_rng(7)
    n = int(np.prod(GRID))
    particles = [rng.uniform(1, 31, (NUM_PARTICLES, 4)).astype(np.float32).tobytes() for _ in range(4)]
    grids = [rng.standard_normal(n).astype(np.float32).tobytes() for _ in range(3)]
    marker = rng.integers(-1, 2, n).astype(np.int8).tobytes()
    pressure = [rng.standard_normal(n).astype(np.float32).tobytes() for _ in range(2)]
    scalars = np.zeros(16, dtype=np.float32).tobytes()  # two 32-byte PCG scalar blocks
    stats = [np.zeros((k, 2), dtype=np.float32).tobytes() for k in NUM_STATS]
    return particles + grids + [marker] + pressure + [scalars] + stats


def state_bytes(**kw):
    hkw = {k: kw[k] for k in ("grid", "max_num_particles", "num_particles", "version", "magic", "num_stats") if k in kw}
    out = header(**hkw)
    for sid, p in enumerate(payloads(), start=1):
        out += section(sid, p)
    return out


def write(tmp_path, data, name="state.blub"):
    p = tmp_path / name
    p.write_bytes(data)
    return str(p)


def info_rc(path):
    L = F.lib()
    out = F.StateInfo()
    rc = L.blub_state_info(os.fsencode(path), out)
    return rc, L.blub_last_error().decode(), out


def test_a_file_written_from_the_documented_layout_is_accepted(tmp_path):
    data = state_bytes()
    n = int(np.prod(GRID))
    assert len(data) == HEADER_BYTES + 13 * 20 + 4 * NUM_PARTICLES * 16 + 5 * n * 4 + n + 64 + 8 * sum(NUM_STATS)
    info = blub_b200.state_info(write(tmp_path, data))
    assert tuple(info.grid_dimension) == GRID
    assert (info.max_num_particles, info.num_particles, info.step_count, info.format_version) == (MAX_PARTICLES, NUM_PARTICLES, STEP_COUNT, 1)


def _flip_payload_byte(data):
    b = bytearray(data)
    b[HEADER_BYTES + 16 + 5] ^= 0x40  # inside the first section's payload (particle positions)
    return bytes(b)


def _section_length_off_by_one(data):
    b = bytearray(data)
    off = HEADER_BYTES
    for _ in range(7):  # skip to the marker section (id 8); its length field says one byte more than the header implies
        length = struct.unpack_from("<Q", b, off + 8)[0]
        off += 16 + length + 4
    assert struct.unpack_from("<I", b, off)[0] == 8
    struct.pack_into("<Q", b, off + 8, struct.unpack_from("<Q", b, off + 8)[0] + 1)
    return bytes(b)


@pytest.mark.parametrize("case,make,needle", [
    ("truncated", lambda: state_bytes()[:-100], "bytes"),
    ("flipped payload byte", lambda: _flip_payload_byte(state_bytes()), "checksum"),
    ("wrong magic", lambda: state_bytes(magic=b"BLUBSTAX"), "magic"),
    ("higher format version", lambda: state_bytes(version=2), "version"),
    ("num_particles above max_num_particles", lambda: state_bytes(max_num_particles=NUM_PARTICLES - 1), "max_num_particles"),
    ("dimension not a multiple of 8", lambda: state_bytes(grid=(32, 36, 40)), "multiples of 8"),
    ("section length disagrees with the header", lambda: _section_length_off_by_one(state_bytes()), "section 8"),
])
def test_malformed_files_are_parse_errors(tmp_path, case, make, needle):
    path = write(tmp_path, make())
    rc, msg, _ = info_rc(path)
    assert rc == BLUB_ERR_PARSE, (case, rc, msg)
    assert needle in msg, (case, msg)
    with pytest.raises(blub_b200.BlubError):
        blub_b200.state_info(path)


def test_header_checksum_covers_the_settings(tmp_path):
    b = bytearray(state_bytes())
    b[80] ^= 0x01  # a bit of the gravity vector
    rc, msg, _ = info_rc(write(tmp_path, bytes(b)))
    assert rc == BLUB_ERR_PARSE and "header checksum" in msg


def test_missing_file_is_an_io_error(tmp_path):
    rc, msg, _ = info_rc(str(tmp_path / "missing.blub"))
    assert rc == BLUB_ERR_IO and "missing.blub" in msg


def test_runner_refuses_to_resume_a_recording_before_touching_a_device(tmp_path):
    runner = os.path.join(os.path.dirname(F.lib_path()), "blub_run")
    res = subprocess.run([runner, util.scene_path("dam_small"), "--load-state", str(tmp_path / "none.blub"), "--record", "30", str(tmp_path / "frame")],
                         capture_output=True, text=True, timeout=60, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert res.returncode == 2, res.stdout + res.stderr
    assert "--record" in res.stderr and not list(tmp_path.iterdir())
