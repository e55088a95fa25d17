"""The direct-call route (EncodeFamilyOf / DecodeFamilyOf in csrc/host_params.cpp, then the block halves
EncodeBlockInterior / DecodeBlockInterior in csrc/kernel_params.h), on the CPU.

tests/native/launch_route_check.cpp compares the route with an independent statement of the tuned launchers' decision
chain -- each launcher checking its description and then its block, and declining the call when either fails -- over
every valid encode and decode description, the context's step-table, Gray16-LUT and verified-shortcut states, and aligned
and misaligned blocks of several sizes (odd 4:2:0 first rows included): same family, same interior, and for the batched
families the same interior in the per-image batch plan."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "avif-format_b200", "csrc")


def test_route_matches_the_launcher_chain(tmp_path):
    exe = tmp_path / "launch_route_check"
    subprocess.run(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-I", "/usr/local/cuda/include", "-I", CSRC,
                    os.path.join(ROOT, "tests", "native", "launch_route_check.cpp"), os.path.join(CSRC, "host_params.cpp"),
                    "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    encode, decode = [dict(re.findall(r"(\w+)=(\d+)", line)) for line in out.stdout.splitlines()[:2]]
    assert int(encode["descriptions"]) > 500 and int(encode["tuned"]) > 10000, out.stdout
    assert int(decode["descriptions"]) > 300 and int(decode["tuned"]) > 10000, out.stdout
