"""Minimal stand-in for the ``detectmatelibrary`` package -- ONLY the two base classes the
reference service imports (``detectmatelibrary.common.core.CoreComponent`` / ``CoreConfig``,
/root/reference/src/service/core.py:20, features/component_loader.py:5,
features/config_loader.py:5, features/config_manager.py:9, features/component_resolver.py:9).

It is put on ``sys.path`` by ``detectmateservice_b200.compat.install_shims()`` only when the
real library cannot be imported (it is not vendored in the reference and not installable
offline), so that this project's components satisfy the loader's ``isinstance(..., CoreComponent)``
check (component_loader.py:52-55) either way.  It contains no detector logic.
"""
__shim__ = True
