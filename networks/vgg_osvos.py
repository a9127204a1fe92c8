"""Import-path shim: ``import networks.vgg_osvos as vo; vo.OSVOS(...)`` keeps working
(reference train_online.py:21,57 / train_parent.py:20,56) and resolves to the H100 implementation."""
from osvos_pytorch_b200.networks.vgg_osvos import OSVOS, he_init_  # noqa: F401
