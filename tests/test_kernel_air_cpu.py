"""The quotient guards of the AIRs whose prover runs hand-written kernels (plonky3_b200.air.KernelAir: the Keccak, Blake3 and
Poseidon2 AIRs), without a GPU: public values, a preprocessed trace or a missing GPU context are refused before any quotient call
reaches the device, and a valid call reaches the AIR's own `Gpu` method with the field, the LDE, the trace height and alpha as
given."""
import numpy as np
import pytest

from plonky3_b200 import _lib
from plonky3_b200.blake3_air import Blake3Air
from plonky3_b200.field import KoalaBear
from plonky3_b200.keccak_air import KeccakAir
from plonky3_b200.poseidon2_air import RoundConstants, VectorizedPoseidon2Air

VEC = 2                    # a Poseidon2 vector length other than the default, so the test sees it passed through


class RecordingGpu:
    """A stand-in device that records every call and answers a quotient call with a token; it computes nothing."""
    device = None

    def __init__(self):
        self.calls = []

    def _record(self, name, args):
        self.calls.append((name, args))
        return ("quotient", name)

    def keccak_air_quotient(self, *args): return self._record("keccak_air_quotient", args)
    def blake3_air_quotient(self, *args): return self._record("blake3_air_quotient", args)
    def p2air_quotient(self, *args): return self._record("p2air_quotient", args)
    def p2air_set_constants(self, *args): self.calls.append(("p2air_set_constants", args))

    def quotient_calls(self):
        return [c for c in self.calls if c[0].endswith("_quotient")]


def _poseidon2(gpu):
    rng = np.random.default_rng(5)
    P = KoalaBear.P
    rc = RoundConstants(rng.integers(0, P, (4, 16)), rng.integers(0, P, 20), rng.integers(0, P, (4, 16)))
    return VectorizedPoseidon2Air(KoalaBear, rc, gpu, vector_len=VEC)


# AIR: (constructor, the name its messages use, its Gpu quotient method, the arguments that method takes after alpha)
AIRS = {
    "keccak": (lambda gpu: KeccakAir(KoalaBear, gpu), "Keccak", "keccak_air_quotient", ()),
    "blake3": (lambda gpu: Blake3Air(KoalaBear, gpu), "Blake3", "blake3_air_quotient", ()),
    "poseidon2": (_poseidon2, "Poseidon2", "p2air_quotient", (VEC,)),
}


@pytest.fixture(scope="module", params=sorted(AIRS))
def kernel_air(request):
    """(name, the AIR built once without a device, its entry in AIRS); each test attaches its own stand-in device."""
    make = AIRS[request.param][0]
    return request.param, make(None), AIRS[request.param]


def _attach(air, gpu):
    air.gpu = gpu
    return air


ALPHA = np.array([3, 5, 7, 11], dtype=np.uint32)


def test_public_values_are_refused(kernel_air):
    _, air, (_, name, _, _) = kernel_air
    gpu = RecordingGpu()
    with pytest.raises(ValueError, match=f"^1 public values given, the {name} AIR has none$"):
        _attach(air, gpu).quotient_values(object(), 4, ALPHA, public_values=[1])
    assert gpu.quotient_calls() == []


def test_a_preprocessed_trace_is_refused(kernel_air):
    _, air, (_, name, _, _) = kernel_air
    gpu = RecordingGpu()
    with pytest.raises(ValueError, match=f"^the {name} AIR has no preprocessed columns$"):
        _attach(air, gpu).quotient_values(object(), 4, ALPHA, preprocessed_on_quotient_domain=object())
    assert gpu.quotient_calls() == []


def test_no_gpu_context_is_refused(kernel_air):
    _, air, _ = kernel_air
    with pytest.raises(_lib.P3GpuError, match="quotient evaluation needs a GPU context"):
        _attach(air, None).quotient_values(object(), 4, ALPHA)


def test_a_valid_call_reaches_the_air_s_own_kernel(kernel_air):
    _, air, (_, _, method, extra) = kernel_air
    gpu = RecordingGpu()
    lde = object()
    q = _attach(air, gpu).quotient_values(lde, 4, ALPHA)
    assert q == ("quotient", method)
    [(called, args)] = gpu.quotient_calls()
    assert called == method and len(args) == 4 + len(extra)
    assert args[0] == KoalaBear.id and args[1] is lde and args[2] == 4 and args[3] is ALPHA and tuple(args[4:]) == extra
