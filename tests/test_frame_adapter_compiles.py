"""CPU: pslam_adapter::ref::FrameConstructor (include/pslam_reference_adapter.hpp) compiles against the reference's headers with the stand-in OpenCV / Eigen /
PCL of oracle/ref/shims, with PSLAM_REF_FULL_HEADERS (the include order of the test libraries: stand-ins first) and without it (the reference tree first, the
way a PlanarSLAM build finds its own headers).  Skipped where the reference tree is absent."""
import os
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"

SRC = r'''
#include <fstream>
#include <iostream>
#include <list>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <sstream>
#include <string>
#include <thread>
#include <vector>
#define protected public
#include "Frame.h"
#include "KeyFrame.h"
#include "Map.h"
#include "MapPoint.h"
#include "MapLine.h"
#include "MapPlane.h"
#include "ORBextractor.h"
#include "Config.h"
#include "KeyFrameDatabase.h"
#undef protected
#include "pslam_reference_adapter.hpp"

// Tracking::GrabImageRGBD's Frame construction, once per frame and for a replayed sequence
void grab(pslam_adapter::ref::FrameConstructor& fc, Planar_SLAM::Frame& F, const cv::Mat& imRGB, const cv::Mat& imGray, const cv::Mat& imDepth, double t,
          Planar_SLAM::ORBVocabulary* voc) {
    fc(F, imRGB, imGray, imDepth, t, voc);
    fc.advance(3);                                  // one MapPlane created
    std::vector<Planar_SLAM::Frame*> fs{&F};
    std::vector<cv::Mat> g{imGray}, d{imDepth};
    fc.batch(fs, g, d, std::vector<double>{t}, voc);
}

pslam_adapter::ref::FrameConstructor* make(Planar_SLAM::ORBextractor* ext, const cv::Mat& K, const cv::Mat& dist) {
    return new pslam_adapter::ref::FrameConstructor(ext, 1000, 1.2f, 8, 20, 7, K, dist, 40.f, 40.f, 1.f / 5000.f, 0.05f, 640, 480, true, 4);
}

int64_t position(const pslam_adapter::ref::FrameConstructor& fc) { return fc.draws() + (int64_t)(fc.call_seconds() + fc.unpack_seconds()); }
'''


def _compile(defines, include_order):
    with tempfile.TemporaryDirectory() as td:
        src = os.path.join(td, "t.cc")
        open(src, "w").write(SRC)
        cmd = ["g++", "-std=gnu++17", "-fsyntax-only", "-w"] + defines + [a for d in include_order for a in ("-I", d)] + ["-I", os.path.join(ROOT, "include"), src]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert r.returncode == 0, r.stdout[-4000:]


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "include")), reason="reference tree absent")
@pytest.mark.parametrize("full", [True, False], ids=["full_headers", "plain"])
def test_frame_constructor_compiles_against_reference_headers(full):
    shims = os.path.join(ROOT, "oracle", "ref", "shims")
    if full:
        _compile(["-DPSLAM_REF_FULL_HEADERS"], [shims, REF, os.path.join(REF, "include")])
    else:
        _compile([], [REF, os.path.join(REF, "include"), shims])
