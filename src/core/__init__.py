"""Drop-in overlay of the reference's `src.core` package (H100 / sm_90a implementations).

Modules this overlay does not provide fall through to the reference's own `src/core` when it
is on sys.path after this repository: the package path is extended over every `src/core`
directory of the `src` namespace package.
"""
import pkgutil

__path__ = pkgutil.extend_path(__path__, __name__)
