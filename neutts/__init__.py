"""Public name of the reference package (`from neutts import NeuTTS`), served by the H100 build.

The class lives in :mod:`neutts.neutts`; everything below its two inner seams is ``libneutts_b200.so``
(see INTEGRATION.md)."""
from neutts.neutts import NeuTTS  # noqa: F401  (re-export)

__all__ = ("NeuTTS",)
