"""`python -m denseflow_b200 <video | folder | list.txt> [-o=.] [-a=tvl1] [-s=0] [-b=32] ...`: see denseflow_b200/cli.py."""
import sys

from .cli import main

sys.exit(main())
