"""Extracts what the tests need from a checkout of the reference repository (ashrafgt/k8s-gpu-hpa):
the container `command:` and `image:` of its Deployment (cuda-test-deployment.yaml:18-19) into
tests/golden/reference_command.json, and the HPA / exporter / scrape settings the offline replay
restates into tests/golden/reference_manifests.json.  The reference is not needed to run the
tests: the parsed values are committed as fixtures.

    python tests/golden/make_reference_command.py <path to the reference checkout>
"""
import json
import os
import re
import sys

import yaml

HERE = os.path.dirname(os.path.abspath(__file__))


def parse(ref: str) -> dict:
    doc = yaml.safe_load(open(os.path.join(ref, "cuda-test-deployment.yaml")))
    c = doc["spec"]["template"]["spec"]["containers"][0]
    return {"source": "cuda-test-deployment.yaml:18-19", "container": c["name"], "image": c["image"], "command": c["command"],
            "gpu_limit": c["resources"]["limits"]["nvidia.com/gpu"]}


def parse_manifests(ref: str) -> dict:
    hpa = open(os.path.join(ref, "cuda-test-hpa.yaml")).read()
    dcgm = open(os.path.join(ref, "dcgm-exporter.yaml")).read().replace("'", '"')
    prom = open(os.path.join(ref, "kube-prometheus-stack-values.yaml")).read()
    num = lambda key: int(re.search(rf"{key}:\s*(\d+)", hpa).group(1))      # noqa: E731
    return {"source": {"hpa": "cuda-test-hpa.yaml:11-12,21", "dcgm": "dcgm-exporter.yaml:37", "prometheus": "kube-prometheus-stack-values.yaml:5"},
            "hpa": {"minReplicas": num("minReplicas"), "maxReplicas": num("maxReplicas"), "targetValue": num("targetValue")},
            "dcgm_collect_interval_ms": int(re.search(r'"-c",\s*"(\d+)"', dcgm).group(1)),
            "scrape_interval": re.search(r"scrape_interval:\s*(\S+)", prom).group(1)}


if __name__ == "__main__":
    ref = sys.argv[1]
    for name, d in (("reference_command.json", parse(ref)), ("reference_manifests.json", parse_manifests(ref))):
        json.dump(d, open(os.path.join(HERE, name), "w"), indent=1)
        print(open(os.path.join(HERE, name)).read())
