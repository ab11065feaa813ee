#!/usr/bin/env python3
"""Regenerates tests/golden/cameras.txt from a checkout of the original project ($CASSIE_REFERENCE); the tests use the committed file and need no
checkout.

  cameras.txt   per model and <camera>: name, body name, pos, quat, fovy (degrees, default 45) and mode (fixed 0, track 1, trackcom 2,
                targetbody 3, targetbodycom 4).  The quaternion comes from the oracle compiler's orientation() (oracle/mjcf_compile.py), an
                implementation independent of the product compiler's (csrc/mjcf.cpp), whose table entries the tests compare with it.
"""
import os
import sys
import xml.etree.ElementTree as ET

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(REPO, 'oracle'))
import mjcf_compile as mc  # noqa: E402

REF = os.environ.get('CASSIE_REFERENCE', '')
MODELS = ['cassie', 'cassie_hfield', 'cassie_tray_box', 'cassie_no_grav', 'cassie_mass', 'cassie_depth']
CAMERA_MODES = dict(fixed=0, track=1, trackcom=2, targetbody=3, targetbodycom=4)


def camera_rows(xml):
    """(name, body name, pos[3], quat[4], fovy, mode) of every <camera> of an MJCF file, in document order"""
    rows = []

    def walk(node, body):
        for c in node:
            if c.tag == 'camera':
                pos = mc.fl(c.get('pos', '0 0 0'))
                rows.append((c.get('name'), body, pos, mc.orientation(c.attrib), float(c.get('fovy', '45')), CAMERA_MODES[c.get('mode', 'fixed')]))
        for c in node:
            if c.tag == 'body':
                walk(c, c.get('name'))
    walk(ET.parse(xml).getroot().find('worldbody'), 'world')
    return rows


def main(path=os.path.join(HERE, 'cameras.txt')):
    assert REF, 'set CASSIE_REFERENCE to a checkout of the original project'
    with open(path, 'w') as f:
        f.write('# model camera body pos[3] quat[4] fovy mode (tests/golden/make_cameras.py)\n')
        for name in MODELS:
            for cam, body, pos, quat, fovy, mode in camera_rows(os.path.join(REF, 'model', name + '.xml')):
                f.write(' '.join([name, cam, body] + [repr(float(x)) for x in list(pos) + list(quat)] + [repr(fovy), str(mode)]) + '\n')
    print('wrote cameras.txt')


if __name__ == '__main__':
    main()
