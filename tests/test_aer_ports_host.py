"""CPU test of Plugin::aerPortHealth's start-up check: the setting is refused, naming it, while aerHealth is off."""
import aer_host as AH
import aer_ports_host as H
import dra_host as DH
import fake_sysfs
import pytest


@pytest.fixture
def hp(tmp_path):
    base, _ = H.make_tree(str(tmp_path))
    p = fake_sysfs.HostPlugin(type("NoGpu", (), {"ctx": None})(), base, str(tmp_path / "pci.ids"), str(tmp_path) + "/")
    DH.configure(p, classes=H.CLASS)
    try:
        yield p
    finally:
        p.close()


def test_refused_without_aer_health(hp):
    H.enable(hp)
    AH.enable(hp, False)
    assert DH.initiate(hp) == "aerPortHealth is set but aerHealth is off"
