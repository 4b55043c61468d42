"""H100-native Flash Checkpoint (see DESIGN.md)."""

import os as _os

if _os.getenv("DLROVER_B200_WIRE_COMPAT", "") in ("1", "true", "True"):
    from . import compat as _compat

    _compat.enable_wire_compat()
