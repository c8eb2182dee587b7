#!/usr/bin/env python
"""in-silico PCR over every primer combination of a multiplex set (multiprime_b200/primer_specificity.py)"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from multiprime_b200.primer_specificity import main  # noqa: E402

if __name__ == "__main__":
    main()
