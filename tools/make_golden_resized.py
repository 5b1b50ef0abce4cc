"""Golden scene for furn_size_rand: Sawyer + table_lack_0825 composed from the MJCF asset tree at the size factor the reference draws for
seed 77 and furn_size_rand = 0.1 (the first draw of RandomState(77), furniture.py:1989-1991), compiled by mjcf.  Needs the asset tree
(FURNITURE_ASSETS); writes tests/golden/Sawyer_table_lack_0825_resized.npz, which lets the test run where the asset tree is absent."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
from furniture_b200 import mjcf  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden", "Sawyer_table_lack_0825_resized.npz")


def main():
    factor = 1 + np.random.RandomState(77).uniform(-0.1, 0.1, 1)[0]
    mjcf.load_scene("Sawyer", "table_lack_0825", resize_factor=factor).save(OUT)
    print("wrote", OUT, "factor", factor)


if __name__ == "__main__":
    main()
