"""Place the unmodified reference (maciejkula/spotlight, pure Python) under
oracle/_ref so that bench.py can time its CPU fit() loop (`--impl reference` and
the `cpu_baseline` entry).  The reference checkout is read from DEFAULT_SRC, or
from the directory the SPOTLIGHT_REFERENCE environment variable names.  Where
neither oracle/_ref nor a checkout exists, install() says so on stderr and the
bench falls back to the restatement in oracle/torch_port.py, which its JSON line
reports as kind "port".  oracle/_ref is a build product and stays out of version
control."""

import os
import shutil
import sys

REF_DST = os.path.join(os.path.dirname(os.path.abspath(__file__)), '_ref')
DEFAULT_SRC = '/root/reference'         # read-only reference checkout of the build environment


def install(src=None):
    """Copy the reference's `spotlight` package into oracle/_ref; return whether it is there."""
    if os.path.isdir(os.path.join(REF_DST, 'spotlight')):
        return True
    src = src or os.environ.get('SPOTLIGHT_REFERENCE') or DEFAULT_SRC
    if not os.path.isdir(os.path.join(src, 'spotlight')):
        sys.stderr.write('oracle/build_ref.py: no reference checkout at %s (set SPOTLIGHT_REFERENCE); '
                         'bench.py will time the oracle/torch_port.py restatement instead\n' % src)
        return False
    shutil.copytree(os.path.join(src, 'spotlight'), os.path.join(REF_DST, 'spotlight'),
                    ignore=shutil.ignore_patterns('__pycache__', '*.pyc'))
    return True
