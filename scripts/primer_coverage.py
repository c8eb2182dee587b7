#!/usr/bin/env python
"""in-silico PCR of a primer set with mismatches on both strands (multiprime_b200/primer_coverage.py)"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from multiprime_b200.primer_coverage import main  # noqa: E402

if __name__ == "__main__":
    main()
