"""Stub so the read-only allRank reference can be imported without its optional cloud / logging dependencies
(only used by the oracle and the tests; never by the product)."""


class GCSFileSystem:
    def open(self, *a, **k):
        raise RuntimeError("gcsfs stub: gs:// paths are not available")
