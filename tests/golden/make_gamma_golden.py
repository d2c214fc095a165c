"""Writes tests/golden/ref_pin_gamma.npz from the REFERENCE's own code (oracle/_ref, oracle/gamma.mk, built where the reference sources are present).
Run from the repo root:  python tests/golden/make_gamma_golden.py

  ref_pin_gamma.npz   what the reference's PhotometricUndistorter, FullSystem::setGammaFunction, FrameHessian::makeImages with that CalibHessian, the PixelSelector and
                      CoarseInitializer::setFirstFromLidar returned in tests/test_ref_pin_gamma.py (tests/ref_golden.py); re-recording gives the same file contents
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))


def main():
    path = os.path.join(HERE, "ref_pin_gamma.npz")
    if os.path.exists(path):
        os.remove(path)                                                      # RefPin.save merges into an existing file: start from none
    env = dict(os.environ, SDV_RECORD_REF_GOLDEN="1")
    subprocess.check_call([sys.executable, "-m", "pytest", "-q", os.path.join(ROOT, "tests", "test_ref_pin_gamma.py")], cwd=ROOT, env=env)


if __name__ == "__main__":
    main()
