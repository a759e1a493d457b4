// TEST INFRASTRUCTURE ONLY -- shared prologue of oracle/ref_store_shim.cpp and oracle/ref_engine_shim.cpp.
// Pulls the reference's OWN sources (read in place from a Wukong checkout, never copied) on top of the std-based stand-ins
// for Boost / TBB / ZeroMQ in oracle/ref_stubs/ (see ref_stubs/README.md).  The stand-ins and the standard library are
// included first, so that the access hack below only opens the reference's own classes.
#pragma once
#include <cmath>
#include <omp.h>
#include <algorithm>
#include <atomic>
#include <fstream>
#include <functional>
#include <iostream>
#include <map>
#include <mutex>
#include <queue>
#include <set>
#include <sstream>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>
// third-party stand-ins first, so that the access hack below only touches the reference's own classes
#include <boost/archive/binary_iarchive.hpp>
#include <boost/algorithm/string.hpp>
#include <boost/archive/binary_oarchive.hpp>
#include <boost/archive/text_oarchive.hpp>
#include <boost/functional/hash.hpp>
#include <boost/mpi.hpp>
#include <boost/serialization/common.hpp>
#include <boost/unordered_map.hpp>
#include <boost/unordered_set.hpp>
#include <boost/variant.hpp>
#include <tbb/concurrent_hash_map.h>
#include <tbb/concurrent_unordered_map.h>
#include <tbb/concurrent_queue.h>
#include <tbb/concurrent_unordered_set.h>
#include <zmq.hpp>
#include <regex>
#include <stdexcept>

#define private public
#define protected public
#include "mem.hpp"
#include "store/static_gstore.hpp"
#ifdef WK_REF_WITH_ENGINE
// core/query.hpp:450 reads `int set_attr_col_num(int n) { attr_col_num = n; }`: a value-returning function without a return
// statement, called by every final_process.  GCC >= 8 compiles that into a trap (-O0) or lets control run off its end (-O1+).
// Without touching the file, give the compiler a well-formed definition: while query.hpp is being read, the declarator
// expands to a complete function followed by the head of a never-called one that swallows the original body.
#define set_attr_col_num(decl) set_attr_col_num(decl) { attr_col_num = n; return 0; } int wk_ref_unused_set_attr_col_num(decl)
#include "query.hpp"
#undef set_attr_col_num
#include "engine/sparql.hpp"   // the reference's SPARQLEngine; dgraph / bind / adaptor / string_server are shadowed (ref_stubs/)
#include "planner.hpp"         // the reference's Planner (only set_plan / set_direction are exercised)
#include "config.hpp"          // the reference's load_config / reload_config (ref_engine_shim.cpp: refc_load_config)
#endif
#undef private
#undef protected


struct RefStore {
    Mem *mem = nullptr;
    StaticGStore *g = nullptr;
    std::vector<uint64_t> segs;   // flattened: index, dir, pid, num_keys, num_buckets, bucket_start, num_edges, edge_start, n_ext, ext0_start, ext0_num
};
