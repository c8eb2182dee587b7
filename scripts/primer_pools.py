#!/usr/bin/env python
"""split a multiplex primer set into balanced pools with the fewest cross products and dimers
(multiprime_b200/primer_pools.py)"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from multiprime_b200.primer_pools import main  # noqa: E402

if __name__ == "__main__":
    main()
