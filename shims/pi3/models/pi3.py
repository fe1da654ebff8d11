"""``from pi3.models.pi3 import Pi3`` (VSLAM/thirdparty/Pi3/pi3/models/pi3.py:17) resolved to the sm_90a implementation."""
from artdeco_b200.pi3 import Pi3  # noqa: F401
