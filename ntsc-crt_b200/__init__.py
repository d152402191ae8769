"""ntsc-crt_b200 -- H100-native composite modulate/demodulate hot path of NTSC-CRT.

The directory name carries a hyphen (it is the project name); import it through
`pkgload.load()` at the repo root, which registers it as module `ntsc_crt_b200`.

Contents (only what the hot path needs):
  csrc/      hand-written sm_90a CUDA kernels + the C-ABI (crt_* drop-in, crtx_* batch)
  lib/       the built shared libraries, one per reference variant (git-ignored)
  layout.py  ctypes mirror of struct CRT / struct NTSC_SETTINGS
  capi.py    loader for the product libraries (fails loudly if they are missing)
"""
import os

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_DIR = os.environ.get("CRT_B200_LIB_DIR") or os.path.join(PKG_DIR, "lib")  # (the override is for debug builds, tools/phase_clocks.py)
CSRC_DIR = os.path.join(PKG_DIR, "csrc")
REPO_ROOT = os.path.dirname(PKG_DIR)

__version__ = "0.1.0"
