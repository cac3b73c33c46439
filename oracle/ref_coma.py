"""TEST / BENCH INFRASTRUCTURE ONLY -- the reference's COMA loss (ding/rl_utils/coma.py), unmodified.

``build()`` byte-compiles that file into ``oracle/_ref/ding_coma.zip`` (git-ignored build output, next to the archives of
``oracle/make_ref.py`` and ``oracle/ref_lm.py`` and made the same way), so that it travels to a machine without the reference
tree; it is run by ``__graft_entry__.build()`` and is a no-op without the tree.  ``module()`` imports it from that archive
into the ``ding.rl_utils`` package that ``oracle/ref_loader.py`` sets up -- never from the reference tree, so a test runs
what travels -- and takes it out of ``sys.modules`` again on exit.  Its ``generalized_lambda_returns`` is the one of the
loaded ``ding.rl_utils.td``.  Nothing in the product package imports this module."""
import contextlib
import importlib
import io
import os
import py_compile
import sys
import tempfile
import warnings
import zipfile

from oracle import ref_loader

REF_ROOT = os.environ.get("DI_ENGINE_REFERENCE", "/root/reference")
HERE = os.path.dirname(os.path.abspath(__file__))
ARCHIVE = os.path.join(HERE, "_ref", "ding_coma.zip")
FILE = "ding/rl_utils/coma.py"
NAME = "ding.rl_utils.coma"


def tree_available():
    return os.path.isfile(os.path.join(REF_ROOT, FILE))


def available():
    return ref_loader.available() and os.path.isfile(ARCHIVE)


def build(force=False):
    """Byte-compile coma.py into the archive; returns its path (None when neither tree nor archive exists)."""
    if not tree_available():
        return ARCHIVE if os.path.isfile(ARCHIVE) else None
    src = os.path.join(REF_ROOT, FILE)
    if not force and os.path.isfile(ARCHIVE):
        t = os.path.getmtime(ARCHIVE)
        if os.path.getmtime(src) <= t and os.path.getmtime(__file__) <= t:
            return ARCHIVE
    os.makedirs(os.path.dirname(ARCHIVE), exist_ok=True)
    buf = io.BytesIO()
    with zipfile.ZipFile(buf, "w", zipfile.ZIP_DEFLATED) as z, tempfile.TemporaryDirectory() as tmp:
        cfile = os.path.join(tmp, "m.pyc")
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", SyntaxWarning)
            py_compile.compile(src, cfile=cfile, dfile=FILE, doraise=True, optimize=0,
                               invalidation_mode=py_compile.PycInvalidationMode.UNCHECKED_HASH)
        z.write(cfile, FILE[:-3] + ".pyc")
        z.writestr("MANIFEST.txt", "byte code (python %d.%d) of the unmodified reference file:\n%s\n" %
                   (sys.version_info[0], sys.version_info[1], FILE))
    with open(ARCHIVE, "wb") as f:
        f.write(buf.getvalue())
    return ARCHIVE


@contextlib.contextmanager
def module():
    """The reference's ``ding.rl_utils.coma`` module, for the duration of the block."""
    if not available():
        raise RuntimeError("reference COMA loss not available: no archive %s" % ARCHIVE)
    pkg = ref_loader.load()
    extra = os.path.join(ARCHIVE, "ding", "rl_utils")
    saved_path = list(pkg.__path__)
    saved = sys.modules.pop(NAME, None)
    pkg.__path__[:] = [extra]  # only the archive: the tree's coma.py must not be picked up
    try:
        mod = importlib.import_module(NAME)
        pkg.__path__[:] = saved_path
        yield mod
    finally:
        pkg.__path__[:] = saved_path
        if saved is None:
            sys.modules.pop(NAME, None)
        else:
            sys.modules[NAME] = saved
