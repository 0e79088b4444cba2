"""Minimal stand-in for `path.py` (not installed, no network): just what the reference's train.py / utils.py touch."""
import os


class Path(str):
    def __truediv__(self, other):
        return Path(os.path.join(str(self), str(other)))

    def __rtruediv__(self, other):
        return Path(os.path.join(str(other), str(self)))

    def makedirs_p(self):
        os.makedirs(str(self), exist_ok=True)
        return self

    def files(self, pattern=None):
        import fnmatch
        out = [Path(os.path.join(self, f)) for f in sorted(os.listdir(self)) if os.path.isfile(os.path.join(self, f))]
        return [f for f in out if pattern is None or fnmatch.fnmatch(os.path.basename(f), pattern)]

    def dirs(self, pattern=None):
        import fnmatch
        out = [Path(os.path.join(self, f)) for f in sorted(os.listdir(self)) if os.path.isdir(os.path.join(self, f))]
        return [d for d in out if pattern is None or fnmatch.fnmatch(os.path.basename(d), pattern)]

    @property
    def name(self):
        return Path(os.path.basename(str(self)))

    @property
    def stem(self):
        return os.path.splitext(os.path.basename(str(self)))[0]

    def dirname(self):
        return Path(os.path.dirname(str(self)))
