"""CPU test of Plugin::draPcieDomain's start-up checks: a domain that is not a lowercase DNS subdomain of at most 63
bytes, one equal to or under kubernetes.io or k8s.io, and any domain while no passthrough class has a draDriver are
refused before any walk, naming the value."""
import dra_host as DH
import dra_pcie_host as H
import fake_sysfs
import pytest


@pytest.fixture
def hp(tmp_path):
    base = H.make_tree(str(tmp_path))
    p = fake_sysfs.HostPlugin(type("NoGpu", (), {"ctx": None})(), base, str(tmp_path / "pci.ids"), str(tmp_path) + "/")
    DH.configure(p, classes=H.CLASSES, dra=H.DRIVERS)
    try:
        yield p
    finally:
        p.close()


@pytest.mark.parametrize("dom", ["Pcie.example.com", "pcie_example.com", "-a.io", "a..io", "a" * 64,
                                 ("a" * 31 + ".") * 2 + "b", "a.io/x"])
def test_refuses_a_bad_domain(hp, dom):
    H.set_domain(hp, dom)
    assert DH.initiate(hp) == 'draPcieDomain "%s" is not a lowercase DNS subdomain of at most 63 bytes' % dom


@pytest.mark.parametrize("dom,root", [("kubernetes.io", "kubernetes.io"), ("k8s.io", "k8s.io"),
                                      ("pcie.kubernetes.io", "kubernetes.io"), ("x.y.k8s.io", "k8s.io")])
def test_refuses_a_reserved_domain(hp, dom, root):
    H.set_domain(hp, dom)
    assert DH.initiate(hp) == 'draPcieDomain "%s" is reserved: names under %s are the standard attributes\'' % (dom, root)


def test_refuses_without_a_dra_driver(hp):
    DH.configure(hp, dra=["", ""])
    H.set_domain(hp, H.DOMAIN)
    assert DH.initiate(hp) == 'draPcieDomain "%s" is set but no passthrough class has a draDriver' % H.DOMAIN
