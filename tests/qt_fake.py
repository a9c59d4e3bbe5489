"""The three Qt classes path_creator needs, reduced to what the tests look at: the bytes a QPainterPath was read from.

``QByteArray`` is a bytearray with ``resize`` and ``replace``; ``QDataStream(buf) >> path`` stores ``bytes(buf)`` on the path as
``path.stream``; ``QPainterPath`` is a plain object (``stream`` None when nothing was read into it).  ``installed()`` puts them
into ``PyQt6.QtCore`` / ``PyQt6.QtGui`` (on top of oracle/ref_loader's stub when that is loaded) and into the globals of the
given modules, and restores everything when the block ends.
"""
import contextlib
import sys
import types


class QByteArray(bytearray):
    def resize(self, n):
        if n > len(self):
            self.extend(bytes(n - len(self)))
        else:
            del self[n:]

    def replace(self, pos, length, data):
        self[pos:pos + length] = data
        return self


class QPainterPath:
    def __init__(self):
        self.stream = None


class QDataStream:
    def __init__(self, buf):
        self.buf = buf

    def __rshift__(self, path):
        path.stream = bytes(self.buf)
        return self


_NAMES = {"PyQt6.QtCore": {"QByteArray": QByteArray, "QDataStream": QDataStream}, "PyQt6.QtGui": {"QPainterPath": QPainterPath}}
_MISSING = object()


@contextlib.contextmanager
def installed(*modules):
    saved_modules = {}
    saved_attrs = []
    try:
        if "PyQt6" not in sys.modules:
            saved_modules["PyQt6"] = _MISSING
            pkg = types.ModuleType("PyQt6")
            pkg.__path__ = []
            sys.modules["PyQt6"] = pkg
        pkg = sys.modules["PyQt6"]
        for name, attrs in _NAMES.items():
            if name not in sys.modules:
                saved_modules[name] = _MISSING
                sys.modules[name] = types.ModuleType(name)
                saved_attrs.append((pkg, name.split(".")[1], getattr(pkg, name.split(".")[1], _MISSING)))
                setattr(pkg, name.split(".")[1], sys.modules[name])
            for target in (sys.modules[name],) + modules:
                for a, v in attrs.items():
                    saved_attrs.append((target, a, target.__dict__.get(a, _MISSING)))
                    setattr(target, a, v)
        yield
    finally:
        for target, a, v in reversed(saved_attrs):
            if v is _MISSING:
                delattr(target, a)
            else:
                setattr(target, a, v)
        for name in saved_modules:
            sys.modules.pop(name, None)
