"""CPU tests of the undistortion in the look-ahead (mloam_frame_set_next_undistort): the entry point in the header, the library and the
binding, and the adapter's and the shim's wrappers compiled against the stub headers."""
import os
import re
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOL = "mloam_frame_set_next_undistort"
ADAPTER = os.path.join(ROOT, "m-loam_b200", "host", "mloam_adapter.hpp")
SHIM = os.path.join(ROOT, "m-loam_b200", "host", "mloam_shim.hpp")


def _compile(td, name, src, includes=()):
    path = os.path.join(td, name + ".cpp")
    with open(path, "w") as f:
        f.write(src)
    obj = os.path.join(td, name + ".o")
    out = subprocess.run(["g++", "-std=c++14", "-Wall", "-Werror"] + ["-I" + i for i in includes] + ["-c", path, "-o", obj],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-3000:]
    return set(re.findall(r"U (mloam_[a-z0-9_]+)", subprocess.run(["nm", "-C", obj], capture_output=True, text=True).stdout))


def test_header_library_and_binding(mloam):
    with open(os.path.join(ROOT, "include", "mloam_b200.h")) as f:
        header = f.read()
    assert re.search(r"^int mloam_frame_set_next_undistort\(mloam_ctx_t \*ctx, int n_lidars, const double \*pose7\);", header, re.M)
    assert SYMBOL in mloam.ABI_SYMBOLS
    getattr(mloam.lib(), SYMBOL)
    assert callable(getattr(mloam.Context, "frame_set_next_undistort"))


def test_adapter_and_shim_wrappers_compile(mloam):
    """mloam_adapter.hpp's undistortMeasurementsNext compiles against the stub headers next to the calls of Estimator::process and needs
    only exported symbols; mloam_shim.hpp's twin compiles."""
    adapter_src = (
        "#include <Eigen/Dense>\n#include <ceres/ceres.h>\n#include <pcl/point_cloud.h>\n#include <pcl/point_types.h>\n"
        '#include "common/types/type.h"\n#include "reference_types.h"\n'
        f'#include "{ADAPTER}"\n'
        "int adapter_next_use(mloam_ctx_t *ctx, const Pose &pose_rlt_next, const std::vector<Eigen::Quaterniond> &qbl_,\n"
        "                     const std::vector<Eigen::Vector3d> &tbl_, size_t IDX_REF, int ESTIMATE_EXTRINSIC) {\n"
        "  std::vector<Pose> pose_undist = mloam::undistortPoses(pose_rlt_next, qbl_, tbl_);\n"
        "  mloam::undistortMeasurementsNext(ctx, pose_undist, IDX_REF, ESTIMATE_EXTRINSIC);\n"
        "  return (int)pose_undist.size();\n}\n")
    shim_src = (f'#include "{SHIM}"\n'
                "int shim_next_use(mloam_ctx_t *ctx) {\n"
                "  std::vector<Pose> p = mloam::undistortPoses(Pose(), 0, std::vector<Pose>(2), 2);\n"
                "  mloam::undistortMeasurementsNext(ctx, p);\n"
                "  return (int)p.size();\n}\n")
    with tempfile.TemporaryDirectory() as td:
        needed = _compile(td, "adapter_next", adapter_src, [os.path.join(ROOT, "tests", "stubs")])
        assert SYMBOL in needed
        for s in needed:
            getattr(mloam.lib(), s)
        assert SYMBOL in _compile(td, "shim_next", shim_src)
