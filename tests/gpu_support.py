"""What the GPU test modules share.  gypsum_b200 is imported inside, so collection works without the library."""
import numpy as np

from oracle import gypsum_oracle as o


def make_engine(fs, n):
    """An engine at fs samples per second and n samples per millisecond, holding the C/A codes of PRN 1 to 32."""
    from gypsum_b200 import _native

    e = _native.Engine(fs, n)
    e.set_replicas(np.stack([o.ca_code(sv) for sv in range(1, 33)]).astype(np.uint8))
    return e
