"""`simple_knn._C.distCUDA2` implemented by libb200gsr.so (dreamscene_b200/csrc/knn.cu)."""
import torch

from dreamscene_b200 import _lib


def distCUDA2(points: torch.Tensor) -> torch.Tensor:
    """points: CUDA float tensor [P,3] -> float32[P], mean squared distance to the 3 nearest other points."""
    if points.device.type != "cuda":
        raise RuntimeError("simple_knn.distCUDA2 (b200gsr): points must be a CUDA tensor; there is no CPU fallback")
    pts = _lib.prepare(points.detach())
    P = int(pts.shape[0])
    out = torch.empty(P, dtype=torch.float32, device=pts.device)
    if P == 0:
        return out
    lib = _lib.load()
    nbytes = int(lib.b200gsr_dist2_scratch_bytes(P))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=pts.device)
    with torch.cuda.device(pts.device):     # the library launches on the CURRENT device
        rc = lib.b200gsr_dist2_knn3(P, _lib.ptr(pts), _lib.ptr(out), _lib.ptr(scratch), nbytes, _lib.stream(pts.device))
    _lib.check(rc, "b200gsr_dist2_knn3")
    return out
