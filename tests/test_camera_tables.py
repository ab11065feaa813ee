"""Camera entries of the compiled model tables (cassie_batch_set_camera).

The product compiler (csrc/mjcf.cpp) records every <camera> as the optional entries names_camera, camera_body[], camera_pos[3 .], camera_quat[4 .],
camera_fovy[] and camera_mode[].  They are checked against tests/golden/cameras.txt, written from the MJCF by the oracle compiler's own orientation
parser (tests/golden/make_cameras.py), with body ids resolved through names_body; with the original project's checkout present, the fixture is also
checked against the MJCF itself."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, REFERENCE, REPO, have_reference
from raycast_support import load_table

MODELS = os.path.join(REPO, 'cassie-mujoco-sim_b200', 'models')
ALL = ('cassie', 'cassie_hfield', 'cassie_tray_box', 'cassie_no_grav', 'cassie_mass', 'cassie_depth')


def fixture():
    rows = {}
    for ln in open(os.path.join(GOLDEN, 'cameras.txt')):
        if not ln.startswith('#'):
            t = ln.split()
            rows.setdefault(t[0], []).append((t[1], t[2], [float(x) for x in t[3:6]], [float(x) for x in t[6:10]], float(t[10]), int(t[11])))
    return rows


@pytest.mark.parametrize('model', ALL)
def test_camera_entries_match_the_fixture(model):
    c, want = load_table(os.path.join(MODELS, model + '.cmodel')), fixture()[model]
    assert c['names_camera'] == [w[0] for w in want]
    assert [c['names_body'][int(b)] for b in c['camera_body']] == [w[1] for w in want]
    assert np.abs(c['camera_pos'] - np.concatenate([w[2] for w in want])).max() <= 1e-15
    assert np.abs(c['camera_quat'] - np.concatenate([w[3] for w in want])).max() <= 1e-15
    assert list(c['camera_fovy']) == [w[4] for w in want] and [int(m) for m in c['camera_mode']] == [w[5] for w in want]


def test_every_model_has_a_camera_and_the_depth_models_a_fixed_one():
    rows = fixture()
    assert all(rows.get(m) for m in ALL)
    for m in ('cassie_depth', 'cassie_hfield'):
        assert ('egocentric', 'cassie-pelvis') in [(r[0], r[1]) for r in rows[m] if r[5] == 0]


def test_depth_table_roundtrip(tmp_path):
    """load_cmodel(save_cmodel(m)) reproduces a table with camera entries byte for byte"""
    src = os.path.join(MODELS, 'cassie_hfield.cmodel')
    subprocess.check_call([sys.executable, os.path.join(REPO, 'tools', 'compile_model.py'), src, str(tmp_path / 'a.cmodel')])
    assert open(src).read() == open(str(tmp_path / 'a.cmodel')).read()


@pytest.mark.skipif(not have_reference(), reason='reference checkout not present')
def test_fixture_is_the_mjcf():
    sys.path.insert(0, os.path.join(REPO, 'tests', 'golden'))
    import make_cameras as mg
    for m, rows in fixture().items():
        got = mg.camera_rows(os.path.join(REFERENCE, 'model', m + '.xml'))
        assert [(r[0], r[1], list(r[2]), list(r[3]), r[4], r[5]) for r in got] == rows, m
