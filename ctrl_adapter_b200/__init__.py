"""ctrl_adapter_b200: H100-native (sm_90a) denoising hot path of Ctrl-Adapter.

The package directory is ``ctrl_adapter_b200/`` (``ctrl-adapter_b200`` at the repository root is a symlink to it, kept
for the repository naming).
"""
__version__ = "0.2.0"
