"""In-tree build of the native artefacts (nvcc cross-compiles sm_90a without a GPU).

    memgraph_b200/_build/libmgb200_pagerank.so   C ABI of include/mgb200_pagerank.h (CUDA runtime linked statically)
    memgraph_b200/_build/pagerank.so             drop-in Memgraph query module (mgp_init_module / mgp_shutdown_module)
    memgraph_b200/_build/libmgp_fake_host.so     fake mgp host used by the tests to load query modules without Memgraph
    memgraph_b200/_build/<module>.so             the other query modules (gpu_bfs, katz_centrality, betweenness_centrality,
                                                 weakly_connected_components, bridges, biconnected_components,
                                                 gpu_wsp, cugraph.* including cugraph.hits), same linking
                                                 as pagerank.so

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
                "wcc.cu", "biconnectivity.cu", "wsp.cu", "hits.cu"]
HEADERS = [os.path.join(CSRC, "core.hpp"), os.path.join(CSRC, "bfs_graph.hpp"), os.path.join(CSRC, "rmat.hpp"), os.path.join(CSRC, "sell_stream.cuh"),
           os.path.join(CSRC, "union_find.cuh"),
           os.path.join(INCLUDE, "mgb200_pagerank.h"), os.path.join(INCLUDE, "mgb200_bfs.h"),
           os.path.join(INCLUDE, "mgb200_katz.h"), os.path.join(INCLUDE, "mgb200_personalized.h"), os.path.join(CSRC, "katz_heap.hpp"),
           os.path.join(INCLUDE, "mgp_abi.h"), os.path.join(CSRC, "mgp_module_common.hpp")]

CORE_LIB = os.path.join(OUT, "libmgb200_pagerank.so")
MODULE_LIB = os.path.join(OUT, "pagerank.so")
FAKE_HOST_LIB = os.path.join(OUT, "libmgp_fake_host.so")
BC_HOST_LIB = os.path.join(OUT, "libmgp_bc_host.so")
BFS_MODULE_LIB = os.path.join(OUT, "gpu_bfs.so")
KATZ_MODULE_LIB = os.path.join(OUT, "katz_centrality.so")
BC_MODULE_LIB = os.path.join(OUT, "betweenness_centrality.so")
WCC_MODULE_LIB = os.path.join(OUT, "weakly_connected_components.so")
WCC_HOST_LIB = os.path.join(OUT, "libmgp_wcc_host.so")
EDGE_HOST_LIB = os.path.join(OUT, "libmgp_edge_host.so")
WSP_MODULE_LIB = os.path.join(OUT, "gpu_wsp.so")
WSP_HOST_LIB = os.path.join(OUT, "libmgp_wsp_host.so")


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


def build_module(objs, verbose=False):
    """The drop-in query module: module glue + the same CUDA objects, CUDA runtime static, so that
    dlopen(RTLD_NOW | RTLD_LOCAL) needs nothing but the host's mgp_* symbols (module.cpp:861)."""
    src = os.path.join(CSRC, "pagerank_module.cpp")
    obj = os.path.join(OUT, "pagerank_module.o")
    if _newer(obj, [src] + HEADERS):
        if verbose:
            print("g++ pagerank_module.cpp", flush=True)
        _run([CXX, "-std=c++20", "-O2", "-fPIC", "-fvisibility=hidden", "-I", INCLUDE, "-I", CSRC, "-c", src, "-o", obj])
    if _newer(MODULE_LIB, objs + [obj]):
        _run([NVCC, "-shared", "-cudart", "static", "-o", MODULE_LIB, obj] + objs)


def build_bfs_module(objs, verbose=False):
    """gpu_bfs.so: the breadth-first expansion as a read procedure (same linking rules as pagerank.so)."""
    src = os.path.join(CSRC, "gpu_bfs_module.cpp")
    obj = os.path.join(OUT, "gpu_bfs_module.o")
    if _newer(obj, [src] + HEADERS):
        if verbose:
            print("g++ gpu_bfs_module.cpp", flush=True)
        _run([CXX, "-std=c++20", "-O2", "-fPIC", "-fvisibility=hidden", "-I", INCLUDE, "-I", CSRC, "-c", src, "-o", obj])
    if _newer(BFS_MODULE_LIB, objs + [obj]):
        _run([NVCC, "-shared", "-cudart", "static", "-o", BFS_MODULE_LIB, obj] + objs)


def build_katz_module(objs, verbose=False):
    """katz_centrality.so: static Katz centrality behind the reference module's name and signature."""
    src = os.path.join(CSRC, "katz_centrality_module.cpp")
    obj = os.path.join(OUT, "katz_centrality_module.o")
    if _newer(obj, [src] + HEADERS):
        if verbose:
            print("g++ katz_centrality_module.cpp", flush=True)
        _run([CXX, "-std=c++20", "-O2", "-fPIC", "-fvisibility=hidden", "-I", INCLUDE, "-I", CSRC, "-c", src, "-o", obj])
    if _newer(KATZ_MODULE_LIB, objs + [obj]):
        _run([NVCC, "-shared", "-cudart", "static", "-o", KATZ_MODULE_LIB, obj] + objs)


def build_bc_module(objs, verbose=False):
    """betweenness_centrality.so: exact betweenness centrality behind the reference module's name and signature."""
    src = os.path.join(CSRC, "betweenness_centrality_module.cpp")
    obj = os.path.join(OUT, "betweenness_centrality_module.o")
    if _newer(obj, [src] + HEADERS):
        if verbose:
            print("g++ betweenness_centrality_module.cpp", flush=True)
        _run([CXX, "-std=c++20", "-O2", "-fPIC", "-fvisibility=hidden", "-I", INCLUDE, "-I", CSRC, "-c", src, "-o", obj])
    if _newer(BC_MODULE_LIB, objs + [obj]):
        _run([NVCC, "-shared", "-cudart", "static", "-o", BC_MODULE_LIB, obj] + objs)


def build_wcc_module(objs, verbose=False):
    """weakly_connected_components.so: weakly connected components behind the reference module's name and signature."""
    src = os.path.join(CSRC, "weakly_connected_components_module.cpp")
    obj = os.path.join(OUT, "weakly_connected_components_module.o")
    if _newer(obj, [src] + HEADERS):
        if verbose:
            print("g++ weakly_connected_components_module.cpp", flush=True)
        _run([CXX, "-std=c++20", "-O2", "-fPIC", "-fvisibility=hidden", "-I", INCLUDE, "-I", CSRC, "-c", src, "-o", obj])
    if _newer(WCC_MODULE_LIB, objs + [obj]):
        _run([NVCC, "-shared", "-cudart", "static", "-o", WCC_MODULE_LIB, obj] + objs)


def build_wsp_module(objs, verbose=False):
    """gpu_wsp.so: the weighted shortest path expansion as a read procedure (same linking rules as pagerank.so)."""
    src = os.path.join(CSRC, "gpu_wsp_module.cpp")
    obj = os.path.join(OUT, "gpu_wsp_module.o")
    if _newer(obj, [src] + HEADERS):
        if verbose:
            print("g++ gpu_wsp_module.cpp", flush=True)
        _run([CXX, "-std=c++20", "-O2", "-fPIC", "-fvisibility=hidden", "-I", INCLUDE, "-I", CSRC, "-c", src, "-o", obj])
    if _newer(WSP_MODULE_LIB, objs + [obj]):
        _run([NVCC, "-shared", "-cudart", "static", "-o", WSP_MODULE_LIB, obj] + objs)


BICONNECTIVITY_MODULE_LIBS = {"bridges": os.path.join(OUT, "bridges.so"),
                              "biconnected_components": os.path.join(OUT, "biconnected_components.so")}


def build_biconnectivity_modules(objs, verbose=False):
    """bridges.so / biconnected_components.so: bridges and biconnected components behind the reference modules' names
    and signatures (one source, compiled twice; MGB200_BRIDGES selects the procedure)."""
    src = os.path.join(CSRC, "biconnectivity_modules.cpp")
    for name, lib in BICONNECTIVITY_MODULE_LIBS.items():
        obj = os.path.join(OUT, f"{name}_module.o")
        if _newer(obj, [src] + HEADERS):
            if verbose:
                print(f"g++ biconnectivity_modules.cpp ({name})", flush=True)
            _run([CXX, "-std=c++20", "-O2", "-fPIC", "-fvisibility=hidden",
                  f"-DMGB200_BRIDGES={1 if name == 'bridges' else 0}", "-I", INCLUDE, "-I", CSRC, "-c", src, "-o", obj])
        if _newer(lib, objs + [obj]):
            _run([NVCC, "-shared", "-cudart", "static", "-o", lib, obj] + objs)


CUGRAPH_MODULE_LIBS = {0: os.path.join(OUT, "cugraph.pagerank.so"), 1: os.path.join(OUT, "cugraph.personalized_pagerank.so")}
CUGRAPH_HITS_MODULE_LIB = os.path.join(OUT, "cugraph.hits.so")


def build_cugraph_modules(objs, verbose=False):
    """cugraph.pagerank.so / cugraph.personalized_pagerank.so / cugraph.hits.so: stand-ins for the reference's cuGraph
    PageRank and HITS modules (one source, compiled three times; module name = file stem, so the procedures are
    cugraph.pagerank.get, cugraph.personalized_pagerank.get and cugraph.hits.get)."""
    src = os.path.join(CSRC, "cugraph_modules.cpp")
    variants = [(f"cugraph_module_{p}.o", f"-DMGB200_CUGRAPH_PERSONALIZED={p}", lib, f"personalized={p}")
                for p, lib in CUGRAPH_MODULE_LIBS.items()]
    variants.append(("cugraph_module_hits.o", "-DMGB200_CUGRAPH_HITS=1", CUGRAPH_HITS_MODULE_LIB, "hits"))
    for obj_name, define, lib, label in variants:
        obj = os.path.join(OUT, obj_name)
        if _newer(obj, [src] + HEADERS):
            if verbose:
                print(f"g++ cugraph_modules.cpp ({label})", flush=True)
            _run([CXX, "-std=c++20", "-O2", "-fPIC", "-fvisibility=hidden", define,
                  "-I", INCLUDE, "-I", CSRC, "-c", src, "-o", obj])
        if _newer(lib, objs + [obj]):
            _run([NVCC, "-shared", "-cudart", "static", "-o", lib, obj] + objs)


FAKE_HOST_SRC = os.path.join(REPO, "tests", "mgp_fake_host.cpp")  # test infrastructure: lives with the tests


def build_fake_host(verbose=False):
    src = FAKE_HOST_SRC
    if _newer(FAKE_HOST_LIB, [src] + HEADERS):
        if verbose:
            print("g++ mgp_fake_host.cpp", flush=True)
        _run([CXX, "-std=c++20", "-O2", "-fPIC", "-shared", "-I", INCLUDE, "-o", FAKE_HOST_LIB, src, "-ldl"])


BC_HOST_SRC = os.path.join(REPO, "tests", "mgp_bc_host.cpp")  # the fake host plus BOOLEAN values and edge ids


def build_bc_host(verbose=False):
    if _newer(BC_HOST_LIB, [BC_HOST_SRC, FAKE_HOST_SRC] + HEADERS):
        if verbose:
            print("g++ mgp_bc_host.cpp", flush=True)
        _run([CXX, "-std=c++20", "-O2", "-fPIC", "-shared", "-I", INCLUDE, "-o", BC_HOST_LIB, BC_HOST_SRC, "-ldl"])


WCC_HOST_SRC = os.path.join(REPO, "tests", "mgp_wcc_host.cpp")  # the BOOLEAN host plus an INTEGER-column call


def build_wcc_host(verbose=False):
    if _newer(WCC_HOST_LIB, [WCC_HOST_SRC, BC_HOST_SRC, FAKE_HOST_SRC] + HEADERS):
        if verbose:
            print("g++ mgp_wcc_host.cpp", flush=True)
        _run([CXX, "-std=c++20", "-O2", "-fPIC", "-shared", "-I", INCLUDE, "-o", WCC_HOST_LIB, WCC_HOST_SRC, "-ldl"])


EDGE_HOST_SRC = os.path.join(REPO, "tests", "mgp_edge_host.cpp")  # the INTEGER host plus (node_from, node_to) rows


def build_edge_host(verbose=False):
    if _newer(EDGE_HOST_LIB, [EDGE_HOST_SRC, WCC_HOST_SRC, BC_HOST_SRC, FAKE_HOST_SRC] + HEADERS):
        if verbose:
            print("g++ mgp_edge_host.cpp", flush=True)
        _run([CXX, "-std=c++20", "-O2", "-fPIC", "-shared", "-I", INCLUDE, "-o", EDGE_HOST_LIB, EDGE_HOST_SRC, "-ldl"])


WSP_HOST_SRC = os.path.join(REPO, "tests", "mgp_wsp_host.cpp")  # the base host plus a node / FLOAT / INTEGER call
HITS_HOST_SRC = os.path.join(REPO, "tests", "mgp_hits_host.cpp")  # the BOOLEAN host plus a call with named FLOAT columns
HITS_HOST_LIB = os.path.join(OUT, "libmgp_hits_host.so")


def build_wsp_host(verbose=False):
    if _newer(WSP_HOST_LIB, [WSP_HOST_SRC, FAKE_HOST_SRC] + HEADERS):
        if verbose:
            print("g++ mgp_wsp_host.cpp", flush=True)
        _run([CXX, "-std=c++20", "-O2", "-fPIC", "-shared", "-I", INCLUDE, "-o", WSP_HOST_LIB, WSP_HOST_SRC, "-ldl"])


def build_hits_host(verbose=False):
    if _newer(HITS_HOST_LIB, [HITS_HOST_SRC, BC_HOST_SRC, FAKE_HOST_SRC] + HEADERS):
        if verbose:
            print("g++ mgp_hits_host.cpp", flush=True)
        _run([CXX, "-std=c++20", "-O2", "-fPIC", "-shared", "-I", INCLUDE, "-o", HITS_HOST_LIB, HITS_HOST_SRC, "-ldl"])


def build_all(verbose=False):
    objs = build_core(verbose)
    if os.path.exists(os.path.join(CSRC, "pagerank_module.cpp")):
        build_module(objs, verbose)
    if os.path.exists(FAKE_HOST_SRC):
        build_fake_host(verbose)
    if os.path.exists(os.path.join(CSRC, "gpu_bfs_module.cpp")):
        build_bfs_module(objs, verbose)
    out = {"core": CORE_LIB}
    if os.path.exists(os.path.join(CSRC, "cugraph_modules.cpp")):
        build_cugraph_modules(objs, verbose)
        out["cugraph_pagerank_module"] = CUGRAPH_MODULE_LIBS[0]
        out["cugraph_personalized_pagerank_module"] = CUGRAPH_MODULE_LIBS[1]
        out["cugraph_hits_module"] = CUGRAPH_HITS_MODULE_LIB
    if os.path.exists(os.path.join(CSRC, "katz_centrality_module.cpp")):
        build_katz_module(objs, verbose)
        out["katz_module"] = KATZ_MODULE_LIB
    if os.path.exists(os.path.join(CSRC, "betweenness_centrality_module.cpp")):
        build_bc_module(objs, verbose)
        out["betweenness_centrality_module"] = BC_MODULE_LIB
    if os.path.exists(os.path.join(CSRC, "weakly_connected_components_module.cpp")):
        build_wcc_module(objs, verbose)
        out["weakly_connected_components_module"] = WCC_MODULE_LIB
    if os.path.exists(os.path.join(CSRC, "biconnectivity_modules.cpp")):
        build_biconnectivity_modules(objs, verbose)
        for name, lib in BICONNECTIVITY_MODULE_LIBS.items():
            out[name + "_module"] = lib
    if os.path.exists(os.path.join(CSRC, "gpu_wsp_module.cpp")):
        build_wsp_module(objs, verbose)
        out["wsp_module"] = WSP_MODULE_LIB
    if os.path.exists(os.path.join(CSRC, "gpu_bfs_module.cpp")):
        out["bfs_module"] = BFS_MODULE_LIB
    if os.path.exists(os.path.join(CSRC, "pagerank_module.cpp")):
        out["module"] = MODULE_LIB
    if os.path.exists(FAKE_HOST_SRC):
        out["fake_host"] = FAKE_HOST_LIB
    if os.path.exists(BC_HOST_SRC):
        build_bc_host(verbose)
        out["bc_host"] = BC_HOST_LIB
    if os.path.exists(WCC_HOST_SRC):
        build_wcc_host(verbose)
        out["wcc_host"] = WCC_HOST_LIB
    if os.path.exists(EDGE_HOST_SRC):
        build_edge_host(verbose)
        out["edge_host"] = EDGE_HOST_LIB
    if os.path.exists(WSP_HOST_SRC):
        build_wsp_host(verbose)
        out["wsp_host"] = WSP_HOST_LIB
    if os.path.exists(HITS_HOST_SRC):
        build_hits_host(verbose)
        out["hits_host"] = HITS_HOST_LIB
    return out


if __name__ == "__main__":
    print(build_all(verbose=True))
