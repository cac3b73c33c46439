"""TEST / BENCH INFRASTRUCTURE ONLY -- the reference's ScatterConnection (ding/torch_utils/network/scatter_connection.py),
unmodified, with the two files a test of the ``hpc_rll`` import path needs next to it: network/rnn.py (which imports
``hpc_rll.torch_utils.network.rnn`` when ``ding.enable_hpc_rl`` is set) and network/normalization.py (which rnn.py imports).

``build()`` byte-compiles the three files into ``oracle/_ref/ding_scatter.zip`` (git-ignored build output, made the way
``oracle/ref_coma.py`` makes its archive) so that they travel to a machine without the reference tree; it is run by
``__graft_entry__.build()`` and is a no-op without the tree.  ``network()`` makes ``ding.torch_utils`` a package whose
``network`` subpackage imports from that archive -- never from the tree -- with ``treetensor`` stubbed (rnn.py imports it
at the top), and on exit restores every ``sys.modules`` entry it touched, so that other tests see the plain
``ding.torch_utils`` module that ``oracle/ref_loader.py`` stubs.  Nothing in the product package imports this module."""
import contextlib
import importlib
import io
import os
import py_compile
import sys
import tempfile
import types
import warnings
import zipfile

from oracle import ref_loader

REF_ROOT = os.environ.get("DI_ENGINE_REFERENCE", "/root/reference")
HERE = os.path.dirname(os.path.abspath(__file__))
ARCHIVE = os.path.join(HERE, "_ref", "ding_scatter.zip")
PACKAGE = "ding.torch_utils.network"
DIR = "ding/torch_utils/network"
FILES = [DIR + "/" + f for f in ("scatter_connection.py", "rnn.py", "normalization.py")]
_TOUCHED = ("ding.torch_utils", "treetensor", "treetensor.torch")


def tree_available():
    return all(os.path.isfile(os.path.join(REF_ROOT, f)) for f in FILES)


def available():
    return ref_loader.available() and os.path.isfile(ARCHIVE)


def build(force=False):
    """Byte-compile the three files into the archive; returns its path (None when neither tree nor archive exists)."""
    if not tree_available():
        return ARCHIVE if os.path.isfile(ARCHIVE) else None
    srcs = [os.path.join(REF_ROOT, f) for f in FILES]
    if not force and os.path.isfile(ARCHIVE):
        t = os.path.getmtime(ARCHIVE)
        if all(os.path.getmtime(s) <= t for s in srcs) and os.path.getmtime(__file__) <= t:
            return ARCHIVE
    os.makedirs(os.path.dirname(ARCHIVE), exist_ok=True)
    buf = io.BytesIO()
    with zipfile.ZipFile(buf, "w", zipfile.ZIP_DEFLATED) as z, tempfile.TemporaryDirectory() as tmp:
        for f, src in zip(FILES, srcs):
            cfile = os.path.join(tmp, "m.pyc")
            with warnings.catch_warnings():
                warnings.simplefilter("ignore", SyntaxWarning)
                py_compile.compile(src, cfile=cfile, dfile=f, doraise=True, optimize=0,
                                   invalidation_mode=py_compile.PycInvalidationMode.UNCHECKED_HASH)
            z.write(cfile, f[:-3] + ".pyc")
        z.writestr("MANIFEST.txt", "byte code (python %d.%d) of the unmodified reference files:\n%s\n" %
                   (sys.version_info[0], sys.version_info[1], "\n".join(FILES)))
    with open(ARCHIVE, "wb") as f:
        f.write(buf.getvalue())
    return ARCHIVE


def _stub_treetensor():
    tt = types.ModuleType("treetensor")
    tt.__path__ = []
    tt.torch = types.ModuleType("treetensor.torch")
    sys.modules["treetensor"] = tt
    sys.modules["treetensor.torch"] = tt.torch


@contextlib.contextmanager
def network():
    """The reference's ``ding.torch_utils.network`` package, importing from the archive, for the duration of the block;
    ``importlib.import_module(PACKAGE + '.scatter_connection')`` (or ``.rnn``) inside it loads the reference file."""
    if not available():
        raise RuntimeError("reference ScatterConnection not available: no archive %s" % ARCHIVE)
    ref_loader.load()
    import ding
    saved = {k: v for k, v in sys.modules.items() if any(k == p or k.startswith(p + ".") for p in _TOUCHED)}
    missing = object()
    saved_attr = getattr(ding, "torch_utils", missing)
    try:
        tu = types.ModuleType("ding.torch_utils")
        stub = saved.get("ding.torch_utils")
        if stub is not None:
            tu.__dict__.update({k: v for k, v in vars(stub).items() if not k.startswith("__")})
        tu.__path__ = []
        sys.modules["ding.torch_utils"] = tu
        net = types.ModuleType(PACKAGE)
        net.__path__ = [os.path.join(ARCHIVE, *DIR.split("/"))]
        sys.modules[PACKAGE] = net
        tu.network = net
        _stub_treetensor()
        with warnings.catch_warnings():  # the reference's docstrings hold a few invalid escape sequences
            warnings.simplefilter("ignore", SyntaxWarning)
            yield net
    finally:
        for k in [k for k in sys.modules if any(k == p or k.startswith(p + ".") for p in _TOUCHED)]:
            del sys.modules[k]
        sys.modules.update(saved)
        if saved_attr is missing:
            if hasattr(ding, "torch_utils"):
                delattr(ding, "torch_utils")
        else:
            ding.torch_utils = saved_attr


def scatter_connection():
    """the reference module ``ding.torch_utils.network.scatter_connection``; call inside ``network()``"""
    return importlib.import_module(PACKAGE + ".scatter_connection")
