"""Rangefinder entries of the compiled model tables (cassie_sim_read_rangefinder).

The product compiler (csrc/mjcf.cpp) records each <rangefinder site= cutoff=> as the optional entries rangefinder_site[] / rangefinder_cutoff[]; the
sensor table and its 29-number layout are unchanged, and a table without the entries (every model but cassie_no_grav.xml) is unchanged byte for byte.
The entries are checked against the MJCF's six rangefinders (tests/golden/cassie_no_grav_rangefinders.txt) and against the oracle compiler's site
table (tests/golden/cassie_no_grav.omodel), which names the sites they refer to; with the original project's checkout present, fresh compiles of every
model are compared with the committed tables byte for byte and the entries with the MJCF itself."""
import filecmp
import os
import subprocess
import sys
import xml.etree.ElementTree as ET

import numpy as np
import pytest

from conftest import GOLDEN, REFERENCE, REPO, have_reference
from raycast_support import load_table

MODELS = os.path.join(REPO, 'cassie-mujoco-sim_b200', 'models')
ALL = ('cassie', 'cassie_hfield', 'cassie_tray_box', 'cassie_no_grav', 'cassie_mass', 'cassie_depth')


def fixture():
    rows = [ln.split() for ln in open(os.path.join(GOLDEN, 'cassie_no_grav_rangefinders.txt')) if not ln.startswith('#')]
    return [(name, site, float(cut)) for name, site, cut in rows]


def test_no_grav_entries_match_the_mjcf_and_the_oracle_site_table():
    c, o = load_table(os.path.join(MODELS, 'cassie_no_grav.cmodel')), load_table(os.path.join(GOLDEN, 'cassie_no_grav.omodel'))
    want = fixture()
    assert len(want) == 6
    sites = [int(s) for s in c['rangefinder_site']]
    assert [c['names_site'][s] for s in sites] == [site for _, site, _ in want]
    assert [o['names_site'][s] for s in sites] == [site for _, site, _ in want]   # the same site ids in the oracle compiler's table
    assert list(c['rangefinder_cutoff']) == [cut for *_, cut in want]
    # the sensor table the step kernel reads is the oracle compiler's, unchanged
    assert int(c['nsensor'][0]) == int(o['nsensor'][0])
    for k in ('sensor_type', 'sensor_objid', 'sensor_cutoff'):
        assert np.array_equal(c[k], o[k]), k


def test_other_tables_carry_no_rangefinder_entries():
    for m in ALL:
        if m != 'cassie_no_grav':
            assert 'rangefinder_site' not in load_table(os.path.join(MODELS, m + '.cmodel')), m


def test_no_grav_table_roundtrip(tmp_path):
    """load_cmodel(save_cmodel(m)) reproduces the table with its rangefinder entries byte for byte"""
    src = os.path.join(MODELS, 'cassie_no_grav.cmodel')
    subprocess.check_call([sys.executable, os.path.join(REPO, 'tools', 'compile_model.py'), src, str(tmp_path / 'a.cmodel')])
    assert filecmp.cmp(src, str(tmp_path / 'a.cmodel'), shallow=False)


@pytest.mark.skipif(not have_reference(), reason='reference checkout not present')
def test_fresh_compiles_equal_the_committed_tables(tmp_path):
    for m in ALL:
        out = str(tmp_path / (m + '.cmodel'))
        subprocess.check_call([sys.executable, os.path.join(REPO, 'tools', 'compile_model.py'), os.path.join(REFERENCE, 'model', m + '.xml'), out])
        assert filecmp.cmp(out, os.path.join(MODELS, m + '.cmodel'), shallow=False), m
    root = ET.parse(os.path.join(REFERENCE, 'model', 'cassie_no_grav.xml')).getroot()
    assert [(x.get('name'), x.get('site'), float(x.get('cutoff'))) for x in root.iter('rangefinder')] == fixture()
