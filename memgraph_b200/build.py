"""In-tree build of the native artefacts (nvcc cross-compiles sm_90a without a GPU).

    memgraph_b200/_build/libmgb200_pagerank.so   C ABI of include/mgb200_pagerank.h (CUDA runtime linked statically)
    memgraph_b200/_build/pagerank.so             drop-in Memgraph query module (mgp_init_module / mgp_shutdown_module)
    memgraph_b200/_build/libmgp_fake_host.so     fake mgp host used by the tests to load query modules without Memgraph
    memgraph_b200/_build/<module>.so             the other query modules (gpu_bfs, katz_centrality, betweenness_centrality,
                                                 weakly_connected_components, bridges, biconnected_components,
                                                 gpu_wsp, bipartite_matching, strongly_connected_components,
                                                 cugraph.* including cugraph.hits),
                                                 same linking as pagerank.so

Objects are rebuilt only when a source or header is newer.  `python -m memgraph_b200.build` builds everything.
"""
import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
OUT = os.path.join(PKG, "_build")
INCLUDE = os.path.join(REPO, "include")

NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CXX = os.environ.get("CXX") or shutil.which("g++") or "g++"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC,-fvisibility=hidden",
    "-Xptxas", "-v",
    "-I", INCLUDE, "-I", CSRC,
    "-diag-suppress", "1444",  # cub::TransformInputIterator deprecation notice
]
CUDA_SOURCES = ["pagerank_kernels.cu", "graph_build.cu", "capi.cu", "bfs.cu", "katz.cu", "personalized.cu", "betweenness.cu",
                "wcc.cu", "biconnectivity.cu", "wsp.cu", "hits.cu", "bipartite_matching.cu", "scc.cu"]
HEADERS = [os.path.join(CSRC, "core.hpp"), os.path.join(CSRC, "bfs_graph.hpp"), os.path.join(CSRC, "rmat.hpp"), os.path.join(CSRC, "sell_stream.cuh"),
           os.path.join(CSRC, "union_find.cuh"), os.path.join(CSRC, "undirected_walk.cuh"),
           os.path.join(INCLUDE, "mgb200_pagerank.h"), os.path.join(INCLUDE, "mgb200_bfs.h"),
           os.path.join(INCLUDE, "mgb200_katz.h"), os.path.join(INCLUDE, "mgb200_personalized.h"), os.path.join(CSRC, "katz_heap.hpp"),
           os.path.join(INCLUDE, "mgp_abi.h"), os.path.join(CSRC, "mgp_module_common.hpp")]

CORE_LIB = os.path.join(OUT, "libmgb200_pagerank.so")


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def _run(cmd, log_name=None):
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if log_name:
        with open(os.path.join(OUT, log_name), "w") as f:
            f.write(" ".join(cmd) + "\n" + proc.stdout)
    if proc.returncode != 0:
        sys.stderr.write(proc.stdout)
        raise RuntimeError("build step failed: " + " ".join(cmd))
    return proc.stdout


def build_core(verbose=False):
    os.makedirs(OUT, exist_ok=True)
    objs = []
    for src in CUDA_SOURCES:
        path = os.path.join(CSRC, src)
        obj = os.path.join(OUT, src.replace(".cu", ".o"))
        if _newer(obj, [path] + HEADERS):
            if verbose:
                print("nvcc", src, flush=True)
            _run([NVCC] + NVCC_FLAGS + ["-c", path, "-o", obj], log_name=src + ".ptxas.log")
        objs.append(obj)
    if _newer(CORE_LIB, objs):
        # -fvisibility=hidden + explicit default visibility on the extern "C" API keeps the export list tight
        _run([NVCC, "-shared", "-cudart", "static", "-o", CORE_LIB] + objs + ["-Xlinker", "--no-undefined"])
    return objs


# The query modules: source in csrc/ -> its outputs as (library, extra -D flags, build_all key).  A source with more than
# one output is compiled once per output; the defines select the procedure (module name = library stem, so cugraph.hits.so
# registers cugraph.hits.get).
MODULES = {
    "pagerank_module.cpp": [("pagerank.so", [], "module")],
    "gpu_bfs_module.cpp": [("gpu_bfs.so", [], "bfs_module")],
    "cugraph_modules.cpp": [
        ("cugraph.pagerank.so", ["-DMGB200_CUGRAPH_PERSONALIZED=0"], "cugraph_pagerank_module"),
        ("cugraph.personalized_pagerank.so", ["-DMGB200_CUGRAPH_PERSONALIZED=1"], "cugraph_personalized_pagerank_module"),
        ("cugraph.hits.so", ["-DMGB200_CUGRAPH_HITS=1"], "cugraph_hits_module")],
    "katz_centrality_module.cpp": [("katz_centrality.so", [], "katz_module")],
    "betweenness_centrality_module.cpp": [("betweenness_centrality.so", [], "betweenness_centrality_module")],
    "weakly_connected_components_module.cpp": [("weakly_connected_components.so", [], "weakly_connected_components_module")],
    "biconnectivity_modules.cpp": [("bridges.so", ["-DMGB200_BRIDGES=1"], "bridges_module"),
                                   ("biconnected_components.so", ["-DMGB200_BRIDGES=0"], "biconnected_components_module")],
    "gpu_wsp_module.cpp": [("gpu_wsp.so", [], "wsp_module")],
    "bipartite_matching_module.cpp": [("bipartite_matching.so", [], "bipartite_matching_module")],
    "strongly_connected_components_module.cpp": [("strongly_connected_components.so", [],
                                                  "strongly_connected_components_module")],
}

# The fake mgp hosts the tests load modules through (test infrastructure, so they live with the tests): library ->
# (build_all key, the host source followed by the host sources it #includes, innermost last).
TESTS = os.path.join(REPO, "tests")
HOSTS = {
    "libmgp_fake_host.so": ("fake_host", ["mgp_fake_host.cpp"]),
    "libmgp_bc_host.so": ("bc_host", ["mgp_bc_host.cpp", "mgp_fake_host.cpp"]),  # plus BOOLEAN values and edge ids
    "libmgp_wcc_host.so": ("wcc_host", ["mgp_wcc_host.cpp", "mgp_bc_host.cpp", "mgp_fake_host.cpp"]),  # plus INTEGER columns
    "libmgp_edge_host.so": ("edge_host", ["mgp_edge_host.cpp", "mgp_wcc_host.cpp", "mgp_bc_host.cpp",
                                          "mgp_fake_host.cpp"]),  # plus (node_from, node_to) rows
    "libmgp_wsp_host.so": ("wsp_host", ["mgp_wsp_host.cpp", "mgp_fake_host.cpp"]),  # plus node / FLOAT / INTEGER rows
    "libmgp_hits_host.so": ("hits_host", ["mgp_hits_host.cpp", "mgp_bc_host.cpp",
                                          "mgp_fake_host.cpp"]),  # plus named FLOAT columns
}


def build_module(src, lib, defines, objs, verbose=False):
    """One query module: its glue + the CUDA objects, CUDA runtime static, so that dlopen(RTLD_NOW | RTLD_LOCAL) needs
    nothing but the host's mgp_* symbols (module.cpp:861)."""
    obj = os.path.join(OUT, lib.replace(".so", "_module.o"))
    if _newer(obj, [os.path.join(CSRC, src)] + HEADERS):
        if verbose:
            print("g++", src, *defines, flush=True)
        _run([CXX, "-std=c++20", "-O2", "-fPIC", "-fvisibility=hidden", *defines, "-I", INCLUDE, "-I", CSRC,
              "-c", os.path.join(CSRC, src), "-o", obj])
    if _newer(os.path.join(OUT, lib), objs + [obj]):
        _run([NVCC, "-shared", "-cudart", "static", "-o", os.path.join(OUT, lib), obj] + objs)


def build_host(lib, chain, verbose=False):
    sources = [os.path.join(TESTS, s) for s in chain]
    if _newer(os.path.join(OUT, lib), sources + HEADERS):
        if verbose:
            print("g++", chain[0], flush=True)
        _run([CXX, "-std=c++20", "-O2", "-fPIC", "-shared", "-I", INCLUDE, "-o", os.path.join(OUT, lib), sources[0],
              "-ldl"])


def build_all(verbose=False):
    objs = build_core(verbose)
    out = {"core": CORE_LIB}
    for src, outputs in MODULES.items():
        if os.path.exists(os.path.join(CSRC, src)):
            for lib, defines, key in outputs:
                build_module(src, lib, defines, objs, verbose)
                out[key] = os.path.join(OUT, lib)
    for lib, (key, chain) in HOSTS.items():
        if os.path.exists(os.path.join(TESTS, chain[0])):
            build_host(lib, chain, verbose)
            out[key] = os.path.join(OUT, lib)
    return out


if __name__ == "__main__":
    print(build_all(verbose=True))
