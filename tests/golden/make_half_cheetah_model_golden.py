"""Generate tests/golden/reference_half_cheetah_model.json: the physical parameters of the reference's HalfCheetah
model, read from vendor/mujoco_models/half_cheetah.xml with xml.etree (nothing is executed or copied).
tests/test_half_cheetah.py re-derives every constant of tests/planar_tree_oracle.py::half_cheetah_model() from it.

Run:  python tests/golden/make_half_cheetah_model_golden.py        (needs /root/reference)
"""
import json
import os
import xml.etree.ElementTree as ET

REF = "/root/reference/vendor/mujoco_models/half_cheetah.xml"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_half_cheetah_model.json")

NUMERIC = {"pos", "axis", "range", "fromto", "size", "friction", "damping", "armature", "stiffness", "ctrlrange",
           "solref", "solimp", "solreflimit", "solimplimit", "timestep", "gravity", "gear", "axisangle", "settotalmass"}


def attrs(e):
    return {k: ([float(t) for t in v.split()] if k in NUMERIC else v) for k, v in e.attrib.items()}


def bodies(e, parent, out):
    for b in e.findall("body"):
        out.append(dict(name=b.get("name"), parent=parent, pos=[float(t) for t in b.get("pos").split()],
                        joints=[attrs(j) for j in b.findall("joint")], geoms=[attrs(g) for g in b.findall("geom")]))
        bodies(b, b.get("name"), out)


if __name__ == "__main__":
    root = ET.parse(REF).getroot()
    m = dict(compiler=attrs(root.find("compiler")), option=attrs(root.find("option")),
             default={c.tag: attrs(c) for c in root.find("default")},
             actuators=[attrs(a) for a in root.find("actuator").findall("motor")])
    m["bodies"] = []
    bodies(root.find("worldbody"), None, m["bodies"])
    with open(OUT, "w") as f:
        json.dump(m, f, indent=1, sort_keys=True)
    print("wrote", OUT)
