"""Sphinx configuration: `sphinx-build -b html docs/source docs/_build` (reference: upstream docs/source/conf.py).

The narrative pages are the Markdown files one directory up (included through MyST when it is installed); the API
reference is generated with autodoc, one page per public module like the reference's docs/source/*.rst.
"""

import os
import sys

sys.path.insert(0, os.path.abspath("../.."))

project = "torchft_b200"
author = "torchft_b200 contributors"
extensions = ["sphinx.ext.autodoc", "sphinx.ext.autosummary", "sphinx.ext.napoleon", "sphinx.ext.viewcode"]
try:  # Markdown narrative pages
    import myst_parser  # noqa: F401

    extensions.append("myst_parser")
    source_suffix = {".rst": "restructuredtext", ".md": "markdown"}
except ImportError:
    source_suffix = {".rst": "restructuredtext"}
autosummary_generate = True
autodoc_default_options = {"members": True, "undoc-members": False, "show-inheritance": True}
# the native extensions need a CUDA toolchain to build; the docs must not
autodoc_mock_imports = ["torchft_b200._K", "torchft_b200._C"]
html_theme = "alabaster"
exclude_patterns = ["_build"]
