"""gcc_b200: the THUDM/GCC pretraining hot path on H100 (sm_90a) -- see DESIGN.md."""
import os as _os

# The pretraining step keeps ~25 CUDA streams busy (training, key encoder, weight gradients, three
# batches of sampler / eigensolver size classes).  With the default of 8 hardware work queues
# unrelated streams share a queue and a kernel can sit for a millisecond behind another stream's
# event wait; 32 is the hardware maximum.  Must be set before the CUDA context is created, hence at
# import time (a value chosen by the user wins).
_os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
