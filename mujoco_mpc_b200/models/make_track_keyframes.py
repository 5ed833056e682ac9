#!/usr/bin/env python
"""Fixture generator: parse the <key> elements of the reference's Humanoid Track mocap clips
(mjpc/tasks/humanoid/tracking/keyframes/*.xml, included by tracking/task.xml:143-152 in the order of
tracking.cc:43-54 kMotionLengths) into tests/golden/humanoid_track_keyframes.npz.

The keyframes are reference DATA (1889 CMU mocap frames: 16 mocap-body positions per frame; qpos / qvel only on the
first frame of a clip).  The parsed arrays are a committed fixture so that the task runs without the reference tree;
`models.load("humanoid_track", keyframes_dir=...)` parses the XMLs directly when the directory is available.

usage: python -m mujoco_mpc_b200.models.make_track_keyframes <reference>/mjpc/tasks/humanoid/tracking/keyframes
"""
import os
import sys
import xml.etree.ElementTree as ET

import numpy as np

CLIPS = ["CMU-CMU-02-02_04", "CMU-CMU-87-87_01", "CMU-CMU-88-88_06", "CMU-CMU-88-88_07", "CMU-CMU-88-88_08",
         "CMU-CMU-88-88_09", "CMU-CMU-90-90_19", "CMU-CMU-103-103_08", "CMU-CMU-108-108_13", "CMU-CMU-137-137_40"]
LENGTHS = [121, 154, 115, 78, 145, 188, 260, 279, 39, 510]          # tracking.cc:43-54


def parse_keyframes(dirpath, nq=28, nv=27, nmocap=16):
    """-> dict(mpos [K][3*nmocap], qpos [K][nq] (NaN rows where the key has none), qvel [K][nv], names [K])."""
    mpos, qpos, qvel, names = [], [], [], []
    for clip, length in zip(CLIPS, LENGTHS):
        root = ET.parse(os.path.join(dirpath, clip + "_poses.xml")).getroot()
        keys = root.findall("./keyframe/key")
        if len(keys) != length:
            raise ValueError("%s: %d keys, tracking.cc expects %d" % (clip, len(keys), length))
        for k in keys:
            mp = np.array(k.get("mpos").split(), float)
            if mp.size != 3 * nmocap:
                raise ValueError("bad mpos size in " + clip)
            mpos.append(mp)
            qpos.append(np.array(k.get("qpos").split(), float) if k.get("qpos") else np.full(nq, np.nan))
            qvel.append(np.array(k.get("qvel").split(), float) if k.get("qvel") else np.zeros(nv))
            names.append(k.get("name"))
    return dict(mpos=np.array(mpos), qpos=np.array(qpos), qvel=np.array(qvel), names=np.array(names))


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    d = parse_keyframes(sys.argv[1])
    root = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    out = os.path.join(root, "tests", "golden", "humanoid_track_keyframes.npz")
    np.savez_compressed(out, mpos=d["mpos"].astype(np.float32), qpos=d["qpos"].astype(np.float32),
                        qvel=d["qvel"].astype(np.float32), names=d["names"])
    print(out, d["mpos"].shape, os.path.getsize(out), "bytes")
