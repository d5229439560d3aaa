"""Recipe of ``build()``: places the unmodified reference package (tenpy/tenpy) under ``oracle/_ref/tenpy``, where
``tenpy_b200.dropin.reference_path()`` finds it.  Test infrastructure only: the tests that run the reference's own
drivers on the engine (drop-in, TEBD, QR truncation, checkpoint exchange, shim) need the reference's code, which is not
part of this repository.  The source is the checkout named by ``$TENPY_REFERENCE`` or, by default, the read-only
checkout of the build machine; without one nothing is done and those tests skip.  ``oracle/_ref/`` is ignored by git."""
import os
import shutil

DEFAULT_SOURCE = '/root/reference'
DEST = os.path.join(os.path.dirname(os.path.abspath(__file__)), '_ref')


def source():
    """the reference checkout to install from, or None if there is none readable"""
    src = os.environ.get('TENPY_REFERENCE') or DEFAULT_SOURCE
    try:
        ok = os.path.isfile(os.path.join(src, 'tenpy', '__init__.py')) and os.access(os.path.join(src, 'tenpy'), os.R_OK)
    except OSError:
        ok = False
    return src if ok else None


def install(dest=DEST):
    """copy the reference's ``tenpy`` package into ``dest`` once (kept while present); returns dest or None"""
    target = os.path.join(dest, 'tenpy')
    if os.path.isfile(os.path.join(target, '__init__.py')):
        return dest
    src = source()
    if src is None:
        return None
    tmp = target + '.partial'
    shutil.rmtree(tmp, ignore_errors=True)
    try:
        shutil.copytree(os.path.join(src, 'tenpy'), tmp, ignore=shutil.ignore_patterns('__pycache__', '*.pyc', '*.so', '*.c'))
        os.replace(tmp, target)
    except OSError:
        shutil.rmtree(tmp, ignore_errors=True)
        return None
    return dest
