"""The conv kernels must compile with a real wgmma pipeline: a conv_*_kernel instantiation whose wgmmas ptxas
serialises (C7510 / C7511: not enough registers to keep a group in flight) or that spills runs correctly but slowly,
with no sign at run time.  The check reads the ptxas report the library build keeps, so it costs no extra compile
when the library is up to date."""
from padel_analytics_b200.build import build_lib, ptxas_problems


def test_conv_kernels_have_no_wgmma_serialisation_or_spills():
    build_lib()
    problems = ptxas_problems()
    assert not problems, "\n".join(problems[:20])
