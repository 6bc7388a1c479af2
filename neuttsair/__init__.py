"""Back-compat alias package of the reference (`from neuttsair import NeuTTSAir`), same class as
:class:`neutts.NeuTTS` on the H100 build."""
from neuttsair.neutts import NeuTTSAir  # noqa: F401  (re-export)

__all__ = ("NeuTTSAir",)
