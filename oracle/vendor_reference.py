#!/usr/bin/env python
"""Install the UNMODIFIED reference into oracle/_ref/ (git-ignored; travels with the built tree).

The reference (skycrapers/TecoGAN-PyTorch) is plain Python with no setup.py / pyproject, so
`pip install --target oracle/_ref <reference>` has nothing to build; the install is a file
copy of its importable tree: codes/**/*.py, the experiment YAMLs and the licence.  Weights
(*.pth), data and images are not needed by any arm and are skipped.  Nothing is edited -- the
module stubs the reference needs on this image (SURVEY.md section 9) are applied at import
time by refimport.py, not to the files.

__graft_entry__.build() calls it; it does nothing where no reference checkout exists (TECOGAN_REFERENCE
names the checkout, default /root/reference).
"""
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.environ.get('TECOGAN_REFERENCE', '/root/reference')
DST = os.path.join(ROOT, 'oracle', '_ref')


def vendor(src=SRC, dst=DST, quiet=False):
    if not os.path.isdir(os.path.join(src, 'codes')):
        return False
    n = 0
    for top in ('codes', 'experiments_BD', 'experiments_BI'):
        for dirpath, dirnames, filenames in os.walk(os.path.join(src, top)):
            dirnames[:] = [d for d in dirnames if d not in ('official_metrics', '__pycache__')]
            for fn in filenames:
                if not fn.endswith(('.py', '.yml', '.yaml', '.txt')) and fn != 'LICENSE':
                    continue
                s = os.path.join(dirpath, fn)
                d = os.path.join(dst, os.path.relpath(s, src))
                os.makedirs(os.path.dirname(d), exist_ok=True)
                if not os.path.isfile(d) or open(s, 'rb').read() != open(d, 'rb').read():
                    shutil.copyfile(s, d)
                n += 1
    for fn in ('LICENSE', 'README.md', 'profile.sh', 'test.sh', 'train.sh'):
        if os.path.isfile(os.path.join(src, fn)):
            shutil.copyfile(os.path.join(src, fn), os.path.join(dst, fn))
    if not quiet:
        print(f'vendor_reference: {n} files -> {dst}')
    return True


if __name__ == '__main__':
    ok = vendor()
    sys.exit(0 if ok else 1)
