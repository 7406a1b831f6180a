"""nope_nerf_b200 — H100-native (sm_90a) NoPe-NeRF render + pose-optimisation hot path.

Host-side mirror of the reference's Python surface (SURVEY.md 8(b)) over the C-ABI CUDA
library libnope_nerf_b200.so.  `import nope_nerf_b200.model as mdl` is a drop-in for the
reference's `import model as mdl` on the hot path."""
from . import _lib  # noqa: F401  (raises loudly when the CUDA library is missing)
from . import ops  # noqa: F401
