"""CPU-side test of csrc/launch_chain.cuh, compiled for the host with g++: which kernel of a Q-network learner's stream launches
with programmatic dependent launch (PDL), and what its prologue may fetch before griddepcontrol.wait.

Results are bit-identical with PDL on or off, so no GPU test notices a lost overlap or a widened early fetch (a data race);
this test pins every rule.  The product library is not involved."""
import itertools
import os
import subprocess

import pytest

from conftest import ROOT

HEADER = os.path.join(ROOT, "dqn-based-uav-3d_path_planer_b200", "csrc", "launch_chain.cuh")
KINDS = ["None", "Act", "Env", "Td", "Train", "TrainFusedTd", "Dw", "Adam"]

DRIVER = r"""
#include <cstdio>
#include "launch_chain.cuh"
std::atomic<int> uavrl::g_pdl{1};
using namespace uavrl;
static void show(const char *tag, ChainLaunch c) { printf("%s %d %d %d %d\n", tag, c.pdl, c.early_weights, c.early_rows, c.flags()); }
int main()
{
    for (int on = 0; on < 2; ++on)
        for (int k = kChainNone; k <= kChainAdam; ++k)
            for (int p = kChainNone; p <= kChainAdam; ++p) {
                printf("rule %d %d %d ", k, p, on);
                show("", chain_launch((ChainKernel)k, (ChainKernel)p, on != 0));
            }
    LaunchChain c;
    c.launched(kChainDw);                                   // outside a scope: nothing is recorded
    show("unscoped", c.next(kChainAdam));
    {
        ChainScope outer(c);
        show("first", c.next(kChainTd));                    // the first kernel of a scope launches plainly
        c.launched(kChainAct);
        show("env", c.next(kChainEnv));
        {
            ChainScope inner(c);                            // a nested scope keeps the chain and its state
            show("nested", c.next(kChainEnv));
            c.launched(kChainEnv);
        }
        show("after_nested", c.next(kChainTrainFusedTd));
        g_pdl.store(0);                                     // uavrl_set_pdl(0): plain launches, the state is still kept
        show("pdl_off", c.next(kChainTrainFusedTd));
        c.launched(kChainDw);
        g_pdl.store(1);
        show("pdl_on", c.next(kChainAdam));
        c.launched(kChainNone);
        show("after_plain", c.next(kChainAct));
    }
    show("closed", c.next(kChainDw));
    {
        ChainScope again(c);
        show("reopened", c.next(kChainAdam));
    }
    return 0;
}
"""


def expected(kind, prev, on):
    """(pdl, early weights, early rows): the rules of the Q-network update, act and env step."""
    if not on:
        return False, False, False
    if kind == "Act":
        return prev != "None", prev == "Env", prev == "Adam"
    if kind == "Td":
        return prev != "None", prev in ("Env", "Td"), False
    pdl = {"Env": prev == "Act", "Train": prev == "Td", "TrainFusedTd": prev == "Env", "Dw": True, "Adam": prev == "Dw",
           "None": False}[kind]
    return pdl, False, False


def flags(pdl, ew, er):
    return (1 | (2 if ew else 0) | (4 if er else 0)) if pdl else 0


@pytest.fixture(scope="module")
def driver_output(tmp_path_factory):
    d = tmp_path_factory.mktemp("launch_chain")
    src, exe = d / "driver.cpp", d / "driver"
    src.write_text(DRIVER)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-std=c++17", "-Wall", "-Werror", "-I", os.path.dirname(HEADER), str(src), "-o", str(exe)])
    return subprocess.check_output([str(exe)], text=True).splitlines()


def test_every_rule(driver_output):
    rules = {}
    for line in driver_output:
        f = line.split()
        if f[0] == "rule":
            k, p, on, pdl, ew, er, fl = map(int, f[1:])
            rules[(KINDS[k], KINDS[p], bool(on))] = ((bool(pdl), bool(ew), bool(er)), fl)
    assert len(rules) == 2 * len(KINDS) ** 2
    for kind, prev, on in itertools.product(KINDS, KINDS, (False, True)):
        want = expected(kind, prev, on)
        assert rules[(kind, prev, on)] == (want, flags(*want)), (kind, prev, on)


def test_scopes_and_switch(driver_output):
    got = {f[0]: tuple(int(x) for x in f[1:]) for f in (line.split() for line in driver_output) if f[0] != "rule"}
    plain = (0, 0, 0, 0)
    assert got == {
        "unscoped": plain, "first": plain,
        "env": (1, 0, 0, 1), "nested": (1, 0, 0, 1), "after_nested": (1, 0, 0, 1),
        "pdl_off": plain, "pdl_on": (1, 0, 0, 1), "after_plain": plain,
        "closed": plain, "reopened": plain,
    }
