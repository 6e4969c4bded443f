"""Generates tests/golden/frame_folder_golden.pt by running the REFERENCE'S OWN DummyDataset.__getitem__ clip selection.

    python tests/golden/make_frame_folder_golden.py <reference checkout>      (pixeli99/SVD_Xtend)

From <reference checkout>/train_svd.py it takes, with `ast`, the class `DummyDataset` and executes it unmodified (no source text is
copied into this repository) over a synthetic folder tree: `os.listdir` returns a fixed order for every folder (not sorted, as a
file system may list them) and `Image.open` records the path it is given and stands for a 2 x 4 RGB frame. Python's global
`random` is seeded once; each pick records the folder and the frames the reference opened, or the ValueError it raised for a
folder with too few frames. tests/test_frames_mixed.py holds svd_xtend_b200.video_train.FrameFolderClips.select to these picks.
"""
import ast
import hashlib
import os
import random
import sys
from types import SimpleNamespace

import numpy as np
import torch

BASE = "videos"
SEED = 20261017
SAMPLE_FRAMES = 4
PICKS = 24
# folder -> frame names, both in the fixed listdir order
TREE = {
    "clip_b": ["0003.png", "0001.png", "0000.png", "0002.png", "0005.png", "0004.png"],
    "clip_a": [f"{i:05d}.jpg" for i in (7, 2, 9, 0, 4, 1, 8, 3, 6, 5)],
    "short": ["b.png", "a.png", "c.png"],
    "clip_c": ["frame_10.png", "frame_2.png", "frame_1.png", "frame_11.png", "frame_3.png"],
    "exact": ["3.png", "1.png", "2.png", "0.png"],
}
ORDER = ["clip_b", "short", "clip_a", "exact", "clip_c"]


def listdir(path):
    if path == BASE:
        return list(ORDER)
    return list(TREE[os.path.relpath(path, BASE)])


def extract(ref_file):
    tree = ast.parse(open(ref_file).read(), filename=ref_file)
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "DummyDataset")
    return compile(ast.fix_missing_locations(ast.Module(body=[cls], type_ignores=[])), ref_file, "exec")


class _Frame:
    def __init__(self, path, opened):
        opened.append(path)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False

    def resize(self, size):
        w, h = size
        return np.zeros((h, w, 3), np.uint8)


def main():
    ref_file = os.path.join(sys.argv[1], "train_svd.py")
    opened = []
    ns = dict(os=SimpleNamespace(listdir=listdir, path=os.path), random=random, torch=torch, np=np,
              Image=SimpleNamespace(open=lambda p: _Frame(p, opened)), Dataset=object)
    exec(extract(ref_file), ns)
    ds = ns["DummyDataset"](BASE, width=4, height=2, sample_frames=SAMPLE_FRAMES)
    random.seed(SEED)
    picks = []
    for _ in range(PICKS):
        opened.clear()
        try:
            ds[0]
        except ValueError as e:
            picks.append(dict(error=str(e)))
            continue
        folder = os.path.dirname(opened[0])
        assert all(os.path.dirname(p) == folder for p in opened)
        picks.append(dict(folder=folder, frames=[os.path.basename(p) for p in opened]))
    fixture = dict(reference_file_sha256=hashlib.sha256(open(ref_file, "rb").read()).hexdigest(), base=BASE, seed=SEED,
                   sample_frames=SAMPLE_FRAMES, order=ORDER, tree=TREE, picks=picks)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "frame_folder_golden.pt")
    torch.save(fixture, path)
    print("wrote", path, sum("error" in p for p in picks), "errors of", len(picks))


if __name__ == "__main__":
    main()
