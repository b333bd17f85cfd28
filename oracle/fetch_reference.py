"""Recipe for oracle/_ref: an UNMODIFIED copy of the reference's `code/` tree (NVlabs/neuralrgbd, plus its LICENSE.md).

    python oracle/fetch_reference.py            # also run by __graft_entry__.build()

The reference is pure Python with no setup.py / pyproject.toml, so there is nothing to compile or `pip install
--target`: its "build" is a verbatim copy of its source tree (0.6 MB). The checkout is taken from $NRGBD_REFERENCE (the
directory that holds `code/`), by default /root/reference. oracle/_ref/ is git-ignored - never part of this repository's
history - and is kept as it is when no checkout is found, so a tree built elsewhere carries its copy along. It is used by
  * tests/test_gpu_dropin.py, tests/test_dropin_host.py  (the reference's own modules and test_utils/test_KVNet.py:test
                                                          driven through neuralrgbd_b200.install_as_reference_modules()),
  * bench.py --impl reference / --impl reference-gpu     (the reference's own KVNET.forward, timed beside the engine).
A MANIFEST with the sha256 of every copied file is written next to it so a reader can check nothing was edited.
"""
import hashlib
import json
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
DST = os.path.join(HERE, '_ref')
CODE = os.path.join(DST, 'code')


def source():
    return os.environ.get('NRGBD_REFERENCE', '/root/reference')


def fetch(verbose=True):
    """Refresh oracle/_ref from the reference checkout. Returns whether oracle/_ref/code exists afterwards."""
    src = source()
    if not os.path.isdir(os.path.join(src, 'code')):
        if verbose:
            print('fetch_reference: no reference checkout at %s - keeping %s as it is' % (src, DST))
        return os.path.isdir(CODE)
    tmp = DST + '.tmp'
    shutil.rmtree(tmp, ignore_errors=True)
    shutil.copytree(os.path.join(src, 'code'), os.path.join(tmp, 'code'), ignore=shutil.ignore_patterns('__pycache__', '*.pyc'))
    for f in ('LICENSE.md', 'README.md'):
        if os.path.exists(os.path.join(src, f)):
            shutil.copy(os.path.join(src, f), os.path.join(tmp, f))
    manifest = {}
    for root, _, files in os.walk(tmp):
        for f in sorted(files):
            p = os.path.join(root, f)
            manifest[os.path.relpath(p, tmp)] = hashlib.sha256(open(p, 'rb').read()).hexdigest()
    with open(os.path.join(tmp, 'MANIFEST.json'), 'w') as fh:
        json.dump({'files': manifest}, fh, indent=1, sort_keys=True)
    shutil.rmtree(DST, ignore_errors=True)
    os.rename(tmp, DST)
    if verbose:
        print('fetch_reference: copied %d files to %s' % (len(manifest), DST))
    return True


def code_dir():
    """The reference's code/ directory to run: $NRGBD_REFERENCE_CODE when set, else oracle/_ref/code; '' when neither exists."""
    d = os.environ.get('NRGBD_REFERENCE_CODE') or CODE
    return d if os.path.isdir(d) else ''


if __name__ == '__main__':
    sys.exit(0 if fetch() else 1)
