from .module_srmr import srmr  # noqa: F401

__all__ = ['srmr']
