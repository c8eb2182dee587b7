#!/usr/bin/env python
"""choose a multiplex primer set from a candidate pool by the targets it amplifies
(multiprime_b200/primer_select.py)"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from multiprime_b200.primer_select import main  # noqa: E402

if __name__ == "__main__":
    main()
