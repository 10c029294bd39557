// TEST INFRASTRUCTURE ONLY: the driver of emu_driver.cpp on the emulation with thread-block clusters (cuda_emu_cluster.h),
// plus what only that emulation has: plans whose Four-Step pairs run as one cluster launch (cluster4.cuh), the switch that
// lets the emulated planner see a cluster-capable device, and a self test of the distributed-shared-memory checkers.
// Built by tests/emu/build_cluster.sh into tests/emu/_build/libb200fft_emu_cluster.so, driven by tests/emu/emu_cluster.py.
#include "emu_driver.cpp"

// both launches of a cluster Four-Step pair through the cluster kernel body (FP32 only)
static int emu_run_cluster(PlanGraph& g, PassPlan& pa, PassPlan& pb, void* const* base) {
    b2_cluster_params K{};
    std::vector<float> lutf[2], hif, lof;
    PassPlan* pps[2] = {&pa, &pb};
    b2_pass_params* Ps[2] = {&K.A, &K.B};
    for (int i = 0; i < 2; ++i) {
        PassPlan& pp = *pps[i];
        b2_pass_params& P = *Ps[i];
        P = pp.P;
        const LutSpec& ls = g.luts[pp.lut_id];
        lutf[i] = make_stage_lut<float>(ls.radices.data(), (int)ls.radices.size());
        P.lut = lutf[i].data();
        if (pp.tw_id >= 0) { make_twolevel<float>(g.tws[pp.tw_id].M, P.tw_shift, hif, lof); P.tw_hi = hif.data(); P.tw_lo = lof.data(); }
        P.in = (const unsigned char*)base[pp.in_role] + pp.in_off * 8;
        P.out = (unsigned char*)base[pp.out_role] + pp.out_off * 8;
    }
    K.nseq = pa.cl_nseq;
    return pa.cluster->launch(&K, nullptr) ? 4039 : 0;
}

// emu_exec_plan with the cluster launches: a pair marked `cluster` runs as one launch of the cluster kernel
extern "C" int emu_cluster_exec_plan(const b200fft_desc* d, int inverse, void* buffer, void* input, void* output, int* npasses) {
    PlanGraph g;
    int rc = build_plan(*d, g);
    if (rc != 0) return rc;
    if (inverse == 1 && !g.has_inv) return R_ONLY_FORWARD;
    if (inverse != 1 && !g.has_fwd) return R_ONLY_INVERSE;
    const size_t esz = g.prec == B2_PREC_F64 ? 16 : 8;
    std::vector<unsigned char> temp(g.temp_elems * esz + 16);
    void* base[ROLE_COUNT] = {buffer, temp.data(), input, output, g_emu_kernel};
    std::vector<PassPlan>& list = (inverse == 1) ? g.inv : g.fwd;
    if (npasses) *npasses = (int)list.size();
    for (size_t i = 0; i < list.size(); ++i) {
        if (list[i].cluster && i + 1 < list.size()) {
            if ((rc = emu_run_cluster(g, list[i], list[i + 1], base)) != 0) return rc;
            ++i;
            continue;
        }
        if (list[i].fused && i + 1 < list.size()) {
            if ((rc = emu_run_fused(g, list[i], list[i + 1], base)) != 0) return rc;
            ++i;
            continue;
        }
        if ((rc = emu_run_one(g, list[i], base)) != 0) return rc;
    }
    return 0;
}

// what the emulated device reports to the planner about thread-block clusters (off: the plans of a device without them)
extern "C" void emu_set_cluster_capable(int on) { b2emu::st().cluster_capable = on != 0; }

// the checkers on distributed shared memory, two clusters of two CTAs: every thread writes its own word, then the same word of
// the other CTA.  Mode 0 = a cluster barrier between the two (correct), 1 = no barrier (write-write hazard across CTAs),
// 2 = a store beyond the peer's allocation, 3 = a store to a CTA rank outside the cluster.  Returns hazards (0-1) or oob (2-3).
extern "C" int emu_selftest_cluster_checkers(int mode) {
    b2emu::State& s = b2emu::st();
    s.hazards = 0; s.smem_oob = false;
    b2emu::launch_cluster(4, 2, 32, 32 * sizeof(float), [&](unsigned char* raw) {
        float* sm = reinterpret_cast<float*>(raw);
        const unsigned t = threadIdx.x, peer = (blockIdx.x % 2) ^ 1u;
        B2_SMEM_ST(sm, t, (float)t);
        if (mode != 1) b2emu::cluster_sync();
        const size_t off = mode == 2 ? (32 + t) * sizeof(float) : t * sizeof(float);
        b2emu::dsmem_st(mode == 3 ? 2u : peer, off, 1.0f);
        b2emu::cluster_sync();
        volatile float v = B2_SMEM_LD(sm, t);
        (void)v;
    }, false);
    const int r = mode >= 2 ? (s.smem_oob ? 1 : 0) : s.hazards.load();
    s.hazards = 0; s.smem_oob = false;
    return r;
}
