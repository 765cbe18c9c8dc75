"""detectmateservice_b200 -- the DetectMate detector-stage hot path on H100 (sm_90a).

Scope (DESIGN.md): Engine._run_loop -> Service.process -> NewValueDetector of
ait-detectmate/DetectMateService, rebuilt as CUDA kernels behind a C ABI
(include/dmdetect.h) with a Python host that mirrors the reference's plugin surface.
"""
__version__ = "0.1.0"
