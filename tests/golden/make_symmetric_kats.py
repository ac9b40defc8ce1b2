#!/usr/bin/env python
"""Extract the reference's inline known answers for TransformationEstimationSymmetric into symmetric_kats.json.

Run in the build container (needs the reference sources; the GPU box does not have them, which is why the result is
committed).  Every number is parsed verbatim from Open3D's C++ test source, except the one expression in these
fixtures, std::sqrt(3.0) / 2.0, which is evaluated; each entry records the file:line span it came from.  The parsing
helpers are make_reference_kats.py's.

    python tests/golden/make_symmetric_kats.py
"""
import json
import os
import re

from make_reference_kats import NUM, init_block, line_of, read

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "symmetric_kats.json")


def main():
    rel = "cpp/tests/t/pipelines/registration/TransformationEstimation.cpp"
    t = read(rel)
    s = t.index("TEST_P(TransformationEstimationPermuteDevices, ComputeRMSESymmetric)")
    e = t.index("TEST_P(TransformationEstimationPermuteDevices, ComputeTransformationSymmetric)")
    body = t[s:e]
    inits = re.findall(r"Tensor::Init<double>\((\{\{.*?\}\})", body, flags=re.S)
    rows = [json.loads(re.sub(r"std::sqrt\((" + NUM + r")\)\s*/\s*(" + NUM + r")",
                              lambda mm: repr(float(mm.group(1)) ** 0.5 / float(mm.group(2))),
                              x).replace("{", "[").replace("}", "]")) for x in inits]
    near = [float(v) for v in re.findall(r"correspondences\),\s*(" + NUM + r"), tolerance\)", body)]
    tols = re.search(r"dtype == core::Float32 \? (" + NUM + r") : (" + NUM + r")", body)
    rmse = {"source": f"{rel}:{line_of(t, s)}-{line_of(t, e) - 1}",
            "source_point": rows[0][0], "source_normal": rows[1][0], "target_point": rows[2][0],
            "target_normal": rows[3][0], "expected": near,
            "tol_f32": float(tols.group(1)), "tol_f64": float(tols.group(2))}
    s = e
    e = t.index("}  // namespace tests", s)
    body = t[s:e]
    ma = re.search(r"AngleAxisd\((" + NUM + r"), Eigen::Vector3d\((" + NUM + r"), (" + NUM + r"), (" + NUM + r")\)", body)
    mtr = re.search(r"block<3, 1>\(0, 3\) = Eigen::Vector3d\((" + NUM + r"), (" + NUM + r"), (" + NUM + r")\)", body)
    robust_expected, _, _ = init_block(body, "const core::Tensor robust_expected")
    # in the test's order: robust_expected, source points, source normals, alternating signs, robust source points,
    # robust source normals, robust noise
    inits = [json.loads(x.replace("{", "[").replace("}", "]"))
             for x in re.findall(r"Tensor::Init<double>\(\s*(\{\{.*?\}\})", body, flags=re.S)]
    mk = re.search(r"RobustKernelMethod::\s*(\w+),\s*(" + NUM + r"),\s*(" + NUM + r")\)", body)
    tols = re.search(r"dtype == core::Float32 \? (" + NUM + r") : (" + NUM + r")", body)
    kats = {
        "rmse": rmse,
        "transformation": {
            "source": f"{rel}:{line_of(t, s)}-{line_of(t, e) - 1}",
            "angle": float(ma.group(1)), "axis": [float(ma.group(k)) for k in (2, 3, 4)],
            "translation": [float(mtr.group(k)) for k in (1, 2, 3)],
            "source_points": inits[1], "source_normals": inits[2], "alternating_signs": [r[0] for r in inits[3]],
            "robust_source_points": inits[4], "robust_source_normals": inits[5], "robust_noise": inits[6],
            "robust_kernel": {"method": mk.group(1), "scaling_parameter": float(mk.group(2)),
                              "shape_parameter": float(mk.group(3))},
            "robust_expected": robust_expected,
            "tol_f32": float(tols.group(1)), "tol_f64": float(tols.group(2))}}
    with open(OUT, "w") as f:
        json.dump(kats, f, indent=1)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
