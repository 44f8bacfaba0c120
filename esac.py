"""Drop-in `import esac` for the reference's callers (train_esac.py:7, test_esac.py:3).

The reference builds a C++ extension module named `esac` exporting exactly forward and backward
(code/esac/esac.cpp:513-516).  This shim exposes the same two names, backed by the
CUDA library of this repository (esac_b200/)."""
from esac_b200.api import backward, forward  # noqa: F401

__all__ = ["forward", "backward"]
