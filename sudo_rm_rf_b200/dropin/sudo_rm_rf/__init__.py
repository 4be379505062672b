"""Drop-in overlay package: only the H100-native modules live here.

Every other sub-module of this package (losses, arg parsers, dataset loaders, the other model
families ...) must keep resolving to the reference checkout that sits LATER on ``sys.path``, so the
package path is extended with the same-named directories found there (``pkgutil.extend_path``)."""
import pkgutil as _pkgutil

__path__ = _pkgutil.extend_path(__path__, __name__)
