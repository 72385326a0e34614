"""Every kernel translation unit of the library, compiled alone for sm_90a: ptxas spills nothing to local memory."""
from kernel_tools import ptxas_report


def test_ptxas_reports_no_spills_in_any_kernel_unit(pkg):
    units = [s for s in pkg.build.SOURCES if s.endswith(".cu")]
    assert "probe_kernels.cu" in units
    for unit in units:
        props = ptxas_report(unit)
        assert props, unit
        assert all(v[1:] == (0, 0) for v in props.values()), (unit, props)
