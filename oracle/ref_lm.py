"""TEST / BENCH INFRASTRUCTURE ONLY -- the reference's language-model losses (ding/rl_utils/grpo.py, rloo.py,
log_prob_utils.py), unmodified.

``build()`` byte-compiles those three files into ``oracle/_ref/ding_lm.zip`` (git-ignored build output, next to the archive
of ``oracle/make_ref.py`` and made the same way), so that they travel to a machine without the reference tree; it is run
by ``__graft_entry__.build()`` and is a no-op without the tree.  ``modules()`` imports them into the ``ding.rl_utils``
package that ``oracle/ref_loader.py`` sets up -- from the tree where it is present, else from the archive -- and takes them
out of ``sys.modules`` again on exit, so that an ``install()`` elsewhere in the same process sees only what the classic
loader loaded.  Nothing in the product package imports this module."""
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
ARCHIVE = os.path.join(HERE, "_ref", "ding_lm.zip")
MODULES = ("log_prob_utils", "grpo", "rloo")
FILES = ["ding/rl_utils/%s.py" % m for m in MODULES]


def tree_available():
    return all(os.path.isfile(os.path.join(REF_ROOT, f)) for f in FILES)


def available():
    return ref_loader.available() and (tree_available() or os.path.isfile(ARCHIVE))


def build(force=False):
    """Byte-compile the three files into the archive; returns its path (None when neither tree nor archive exists)."""
    if not tree_available():
        return ARCHIVE if os.path.isfile(ARCHIVE) else None
    if not force and os.path.isfile(ARCHIVE):
        t = os.path.getmtime(ARCHIVE)
        if all(os.path.getmtime(os.path.join(REF_ROOT, f)) <= t for f in FILES) and os.path.getmtime(__file__) <= t:
            return ARCHIVE
    os.makedirs(os.path.dirname(ARCHIVE), exist_ok=True)
    buf = io.BytesIO()
    with zipfile.ZipFile(buf, "w", zipfile.ZIP_DEFLATED) as z, tempfile.TemporaryDirectory() as tmp:
        for rel in FILES:
            cfile = os.path.join(tmp, "m.pyc")
            with warnings.catch_warnings():
                warnings.simplefilter("ignore", SyntaxWarning)
                py_compile.compile(os.path.join(REF_ROOT, rel), cfile=cfile, dfile=rel, doraise=True, optimize=0,
                                   invalidation_mode=py_compile.PycInvalidationMode.UNCHECKED_HASH)
            z.write(cfile, rel[:-3] + ".pyc")
        z.writestr("MANIFEST.txt", "byte code (python %d.%d) of the unmodified reference files:\n%s\n" %
                   (sys.version_info[0], sys.version_info[1], "\n".join(FILES)))
    with open(ARCHIVE, "wb") as f:
        f.write(buf.getvalue())
    return ARCHIVE


@contextlib.contextmanager
def modules():
    """{'grpo': module, 'rloo': module, 'log_prob_utils': module} of the reference, for the duration of the block."""
    if not available():
        raise RuntimeError("reference language-model losses not available: no tree at %s and no archive %s" %
                           (REF_ROOT, ARCHIVE))
    pkg = ref_loader.load()
    extra = None
    if ref_loader.source() != "tree" or not tree_available():
        extra = os.path.join(ARCHIVE, "ding", "rl_utils")
        pkg.__path__.append(extra)
    names = ["ding.rl_utils." + m for m in MODULES]
    saved = {n: sys.modules.get(n) for n in names}
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", SyntaxWarning)
            yield {m: importlib.import_module("ding.rl_utils." + m) for m in MODULES}
    finally:
        for n, mod in saved.items():
            if mod is None:
                sys.modules.pop(n, None)
            else:
                sys.modules[n] = mod
        if extra is not None and extra in pkg.__path__:
            pkg.__path__.remove(extra)
