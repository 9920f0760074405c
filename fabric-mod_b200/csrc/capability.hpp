// Argument checks of fabgpu_channel_capability, fabgpu_namespace_policies and fabgpu_namespace_versions: host code, shared by the shim
// and the tests' host build (tests/host_sim/blockdev_v13.inc).  Each returns null when the call may proceed, else the refusal text.
#pragma once
#include <stdint.h>
#include <vector>
#include "../../include/fabgpu_ecdsa.h"
#include "blockval.hpp"

namespace fabgpu { namespace capability {

// true when a tree from one of `roots` of the configured policy reaches an ImplicitMeta node (fabgpu_msp_configure checked the trees
// acyclic and at most BD_MAX_POLICY_DEPTH deep)
inline bool reaches_implicit_meta(const std::vector<blockval::PolicyNode>& nodes, const int32_t* roots, int n)
{
    std::vector<int32_t> stack(roots, roots + n);
    std::vector<uint8_t> seen(nodes.size(), 0);
    while (!stack.empty()) {
        const int32_t i = stack.back(); stack.pop_back();
        if (i < 0 || i >= (int32_t)nodes.size() || seen[i]) continue;
        seen[i] = 1;
        if (nodes[i].type == 2) return true;
        if (nodes[i].type == 0)
            for (int c = nodes[i].first_child; c < nodes[i].first_child + nodes[i].n_children; c++) stack.push_back(c);
    }
    return false;
}

// The policies a namespace table gives: its roots, or node 0 for every namespace when it is empty.  In v1.3 mode they are lscc chaincode
// definitions, which hold signature policies only.
inline const char* table_for_v13(const std::vector<blockval::PolicyNode>& nodes, const int32_t* ns_root, int n_ns)
{
    const int32_t zero = 0;
    const bool meta = n_ns ? reaches_implicit_meta(nodes, ns_root, n_ns) : !nodes.empty() && reaches_implicit_meta(nodes, &zero, 1);
    return meta ? "a namespace policy reaches an ImplicitMeta node: the v1.3 mode takes signature policies only" : nullptr;
}

// fabgpu_channel_capability(cap) with the namespace table ns_root[0, n_ns) installed
inline const char* check_capability(int cap, const std::vector<blockval::PolicyNode>& nodes, const int32_t* ns_root, int n_ns)
{
    if (cap != FABGPU_CAP_V2_0 && cap != FABGPU_CAP_V1_3) return "channel capability is not FABGPU_CAP_V2_0 or FABGPU_CAP_V1_3";
    return cap == FABGPU_CAP_V1_3 ? table_for_v13(nodes, ns_root, n_ns) : nullptr;
}

// fabgpu_namespace_policies(ns_root, n_ns) in mode v13 (or not); the roots are already checked inside the node array
inline const char* check_namespace_table(bool v13, const std::vector<blockval::PolicyNode>& nodes, const int32_t* ns_root, int n_ns)
{
    return v13 ? table_for_v13(nodes, ns_root, n_ns) : nullptr;
}

// fabgpu_namespace_versions(ver_off, n_ns) with a namespace table of table_n entries
inline const char* check_versions(const uint32_t* ver_off, int n_ns, int table_n)
{
    if (n_ns != table_n) return "namespace versions do not match the installed namespace table";
    for (int i = 0; i < n_ns; i++)
        if (ver_off[i] > ver_off[i + 1]) return "namespace version offsets decrease";
    return nullptr;
}

} }  // namespace fabgpu::capability
