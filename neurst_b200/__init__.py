"""neurst_b200 — H100-native SpeechTransformer hot path (libb200st) behind the bytedance/neurst class registry.

Importing the package registers the H100 classes into the reference's registries when the reference is importable
(`--include neurst_b200` in the reference CLI does exactly this import, neurst/utils/flags_core.py:207-247); without the
reference on sys.path the package is a stand-alone library (models / layers / trainer / decode on top of the C ABI).
"""
__version__ = "0.2.0"


def _try_register():
    import sys
    if "neurst" not in sys.modules and "neurst_pt" not in sys.modules:
        return None        # the reference is not loaded in this process: nothing to plug into
    try:
        from neurst_b200 import plugin
        if plugin.reference_available():
            return plugin.register()
    except Exception:      # a half-importable reference (e.g. TF missing for the tf registries) must not break the library
        return None
    return None


REGISTERED = _try_register()
