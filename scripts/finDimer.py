#!/usr/bin/env python
"""drop-in for the reference's scripts/finDimer.py: same flags and output files, computed by libmpb200 on an H100
(point the Snakemake `scripts_dir` at this directory)"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from multiprime_b200.findimer import main  # noqa: E402

if __name__ == "__main__":
    main()
