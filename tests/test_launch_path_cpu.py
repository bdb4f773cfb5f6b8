"""Every kernel the host layer starts goes through one launch helper (granne_b200.cu: launch), which counts the launch
on its handle and reports a failed launch to the call that made it.  A second launch site would bypass both."""
import os

CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "granne_b200", "csrc", "granne_b200.cu")


def test_one_launch_site():
    assert open(CU).read().count("<<<") == 1
