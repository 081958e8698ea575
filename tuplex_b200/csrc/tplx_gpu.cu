// tplx_gpu.cu — C-ABI implementation (host side of libtplx_gpu.so).
//
// Plays the role of LocalBackend::executeTransformStage + TransformTask for the GPU:
// (reference tuplex/core/src/ee/local/LocalBackend.cc:815-1252, core/src/physical/TransformTask.cc:382-513)
// validates a stage descriptor, keeps device copies of the program, sizes tiles/shared memory,
// launches the stage kernels on a per-device stream, and hands back results in column form, in the
// reference's Partition byte format, and as exception records.
//
// No CPU fallback exists in this file by design: every compute entry point requires a CUDA device.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/tplx_gpu.h"
#include "kernels.cuh"
#include "rowfmt.cuh"
#include "hashagg.cuh"
#include "fused.cuh"
#include "gather.cuh"
#include "mask.cuh"
#include "vecvm.cuh"
#include "csv.cuh"
#include "text.cuh"
#include "join.cuh"
#include "option.cuh"
#include "merge.cuh"
#include "concat.cuh"
#include "cache.cuh"
#include "sort.cuh"
#include "jit.inl"

using namespace tplx;

// ---------------------------------------------------------------------------------------------
// errors
// ---------------------------------------------------------------------------------------------
static thread_local std::string g_last_error;
static int32_t fail(int32_t code, const std::string &msg) {
    g_last_error = msg;
    return code;
}
#define CU(call)                                                                              \
    do {                                                                                      \
        cudaError_t _e = (call);                                                              \
        if (_e != cudaSuccess) {                                                              \
            return fail(TPLX_E_CUDA, std::string(#call) + ": " + cudaGetErrorString(_e));     \
        }                                                                                     \
    } while (0)

extern "C" const char *tplx_gpu_last_error(void) { return g_last_error.c_str(); }

// ---------------------------------------------------------------------------------------------
// devices
// ---------------------------------------------------------------------------------------------
struct Device {
    int id = -1;
    cudaStream_t stream = nullptr;       // compute stream
    cudaStream_t copy_stream = nullptr;  // H2D uploads, so that the next block's copy overlaps this block's kernels
    cudaStream_t d2h_stream = nullptr;   // result fetches: must not queue behind another block's kernels
    cudaDeviceProp prop{};
    int smem_optin = 0;
    uint8_t *scratch = nullptr;
    size_t scratch_bytes = 0;
    uint64_t *pinned = nullptr;  // small page-locked buffer: counts fetched with stream-ordered copies that never block the host
    std::mutex mu;
    Device *alt = nullptr;  // second execution lane on the same GPU (own streams + scratch): lets the kernels of two
                            // blocks overlap (e.g. the latency-bound dense launch of one with the prefilter of the next)
};
static std::vector<Device *> g_devices;
static std::mutex g_mu;

static Device *get_device(int32_t device) {
    for (auto *d : g_devices)
        if (d->id == device) return d;
    return nullptr;
}

extern "C" int32_t tplx_gpu_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

extern "C" int32_t tplx_gpu_init(const int32_t *devices, int32_t n) {
    std::lock_guard<std::mutex> lk(g_mu);
    int count = tplx_gpu_device_count();
    if (count <= 0) return fail(TPLX_E_NODEVICE, "no CUDA device visible; the GPU backend has no CPU fallback");
    std::vector<int32_t> want;
    if (!devices || n <= 0) want.push_back(0);
    else want.assign(devices, devices + n);
    for (int32_t id : want) {
        if (id < 0 || id >= count) return fail(TPLX_E_BADARG, "device index out of range");
        if (get_device(id)) continue;
        Device *d = new Device();
        d->id = id;
        CU(cudaSetDevice(id));
        CU(cudaGetDeviceProperties(&d->prop, id));
        CU(cudaStreamCreateWithFlags(&d->stream, cudaStreamNonBlocking));
        CU(cudaStreamCreateWithFlags(&d->copy_stream, cudaStreamNonBlocking));
        CU(cudaStreamCreateWithFlags(&d->d2h_stream, cudaStreamNonBlocking));
        CU(cudaHostAlloc(&d->pinned, 64 * 8, cudaHostAllocDefault));
        CU(cudaDeviceGetAttribute(&d->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, id));
        cudaMemPool_t pool;
        CU(cudaDeviceGetDefaultMemPool(&pool, id));
        uint64_t thr = UINT64_MAX;
        CU(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr));
        CU(cudaFuncSetAttribute(stage_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, d->smem_optin));
        CU(cudaFuncSetAttribute(stage_agg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, d->smem_optin));
        CU(cudaFuncSetAttribute(stage_hash_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, d->smem_optin));
        CU(cudaFuncSetAttribute(stage_hash_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, d->smem_optin));
        CU(cudaFuncSetAttribute(stage_hash_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, d->smem_optin));
        CU(cudaFuncSetAttribute(stage_mask_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, d->smem_optin));
        CU(cudaFuncSetAttribute(stage_mask_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, d->smem_optin));
        // extra execution lanes on the same GPU (chain d -> alt -> alt ...): two lanes in all let the latency-bound dense
        // launch of one block overlap the prefilter of the next
        constexpr int lanes = 2;
        Device *tail = d;
        for (int l = 1; l < lanes; ++l) {
            Device *a = new Device();
            a->id = id;
            a->prop = d->prop;
            a->smem_optin = d->smem_optin;
            CU(cudaStreamCreateWithFlags(&a->stream, cudaStreamNonBlocking));
            CU(cudaStreamCreateWithFlags(&a->copy_stream, cudaStreamNonBlocking));
            CU(cudaStreamCreateWithFlags(&a->d2h_stream, cudaStreamNonBlocking));
            CU(cudaHostAlloc(&a->pinned, 64 * 8, cudaHostAllocDefault));
            tail->alt = a;
            tail = a;
        }
        g_devices.push_back(d);
    }
    return TPLX_OK;
}

extern "C" int32_t tplx_gpu_shutdown(void) {
    std::lock_guard<std::mutex> lk(g_mu);
    for (auto *d : g_devices) {
        cudaSetDevice(d->id);
        for (Device *a = d->alt; a;) {
            Device *next = a->alt;
            cudaStreamSynchronize(a->stream);
            if (a->scratch) cudaFree(a->scratch);
            cudaStreamDestroy(a->stream);
            cudaStreamDestroy(a->copy_stream);
            cudaStreamDestroy(a->d2h_stream);
            delete a;
            a = next;
        }
        cudaStreamSynchronize(d->stream);
        if (d->scratch) cudaFree(d->scratch);
        cudaStreamDestroy(d->stream);
        cudaStreamDestroy(d->copy_stream);
        cudaStreamDestroy(d->d2h_stream);
        delete d;
    }
    g_devices.clear();
    return TPLX_OK;
}

extern "C" int32_t tplx_gpu_device_info(int32_t device, char *name_buf, int32_t buf_len, int32_t *sm_count,
                                        uint64_t *mem_bytes) {
    Device *d = get_device(device);
    if (!d) return fail(TPLX_E_BADARG, "device not initialised (call tplx_gpu_init)");
    if (name_buf && buf_len > 0) {
        strncpy(name_buf, d->prop.name, buf_len - 1);
        name_buf[buf_len - 1] = 0;
    }
    if (sm_count) *sm_count = d->prop.multiProcessorCount;
    if (mem_bytes) *mem_bytes = d->prop.totalGlobalMem;
    return TPLX_OK;
}

// ---------------------------------------------------------------------------------------------
// stage
// ---------------------------------------------------------------------------------------------
// ---- K1v planner: IR ops of a fixed-width stage -> vector micro-ops (vecvm.cuh) --------------------------------------------------
// Straight-line liveness over slots decides what never has to touch the shared-memory register file:
//   * x % 2^k feeding only an integer compare        -> the compare masks its operand (VX_A_MASK), the modulo disappears;
//   * a boolean op feeding only the next FILTER       -> the op filters (VX_FILTER), the FILTER disappears;
//   * producer immediately followed by its consumer   -> the operand comes from the accumulator (VX_A_ACC / VX_B_ACC);
//   * a result that no later micro-op reads from its slot and that is no output column -> not stored (VX_NOSTORE);
//   * the slots still in use are renumbered densely (fewer slots = more resident CTAs).
// Only unguarded ops take part (a guarded op merges with the old destination and may be skipped by the warp); ops that can
// raise keep operands and result in slots (they run row by row). Semantics per row are untouched: the same single integer /
// IEEE operations in the same order.
struct VecIns {
    tplx_instr in;
    uint32_t vop = V_NOP, xf = 0;
};
struct VecPlan {
    std::vector<VecIns> ins;
    std::vector<uint16_t> slot_map;  // IR slot -> dense slot (TPLX_NOSLOT = unused)
    uint32_t n_slots = 1;
};
static bool vop_raising(uint32_t v) { return v == V_IFLOORDIV || v == V_IMOD || v == V_FDIV || v == V_FMOD || v == V_FFLOORDIV; }
static bool vop_pred(uint32_t v) { return v == V_BAND || v == V_BOR || v == V_BNOT || (v >= V_ICMP_EQ && v <= V_FCMP_GE); }
static bool vop_icmp(uint32_t v) { return v >= V_ICMP_EQ && v <= V_ICMP_GE; }
// operands read: bit 0 = a, bit 1 = b, bit 2 = c (before constant flags)
static uint32_t vop_reads(uint32_t v) {
    switch (v) {
        case V_NOP: case V_LDCOL: case V_LDI: case V_LDROW: case V_RAISE: return 0;
        case V_MOV: case V_INEG: case V_IABS: case V_FNEG: case V_FABS: case V_I2F: case V_F2I: case V_BNOT: case V_ISHRK: case V_IANDK: case V_FILTER: return 1;
        case V_SEL: return 7;
        default: return 3;
    }
}
static bool vop_has_dst(uint32_t v) { return v != V_NOP && v != V_FILTER && v != V_RAISE; }
static VecPlan vec_plan(const std::vector<tplx_instr> &prog, const std::vector<tplx_outcol> &outs, uint32_t n_slots_ir) {
    VecPlan pl;
    for (const tplx_instr &in : prog) {
        VecIns v;
        v.in = in;
        switch (in.op) {
            case TPLX_OP_LDCOL: v.vop = V_LDCOL; break;
            case TPLX_OP_LDI: v.vop = V_LDI; break;
            case TPLX_OP_LDROW: v.vop = V_LDROW; break;
            case TPLX_OP_MOV: v.vop = V_MOV; break;
            case TPLX_OP_SEL: v.vop = V_SEL; break;
            case TPLX_OP_IADD: v.vop = V_IADD; break;
            case TPLX_OP_ISUB: v.vop = V_ISUB; break;
            case TPLX_OP_IMUL: v.vop = V_IMUL; break;
            case TPLX_OP_INEG: v.vop = V_INEG; break;
            case TPLX_OP_IAND: v.vop = V_IAND; break;
            case TPLX_OP_IOR: v.vop = V_IOR; break;
            case TPLX_OP_IXOR: v.vop = V_IXOR; break;
            case TPLX_OP_ISHL: v.vop = V_ISHL; break;
            case TPLX_OP_ISHR: v.vop = V_ISHR; break;
            case TPLX_OP_IABS: v.vop = V_IABS; break;
            case TPLX_OP_FADD: v.vop = V_FADD; break;
            case TPLX_OP_FSUB: v.vop = V_FSUB; break;
            case TPLX_OP_FMUL: v.vop = V_FMUL; break;
            case TPLX_OP_FNEG: v.vop = V_FNEG; break;
            case TPLX_OP_FABS: v.vop = V_FABS; break;
            case TPLX_OP_I2F: v.vop = V_I2F; break;
            case TPLX_OP_F2I: v.vop = V_F2I; break;
            case TPLX_OP_BAND: v.vop = V_BAND; break;
            case TPLX_OP_BOR: v.vop = V_BOR; break;
            case TPLX_OP_BNOT: v.vop = V_BNOT; break;
            case TPLX_OP_ICMP: v.vop = V_ICMP_EQ + std::min<uint32_t>(in.flags & 7, 5); break;
            case TPLX_OP_FCMP: v.vop = V_FCMP_EQ + std::min<uint32_t>(in.flags & 7, 5); break;
            case TPLX_OP_IFLOORDIV: v.vop = V_IFLOORDIV; break;
            case TPLX_OP_IMOD: v.vop = V_IMOD; break;
            case TPLX_OP_FDIV: v.vop = V_FDIV; break;
            case TPLX_OP_FMOD: v.vop = V_FMOD; break;
            case TPLX_OP_FFLOORDIV: v.vop = V_FFLOORDIV; break;
            case TPLX_OP_FILTER: v.vop = V_FILTER; break;
            case TPLX_OP_RAISE: v.vop = V_RAISE; break;
            default: v.vop = V_NOP; break;
        }
        if (v.vop == V_NOP) continue;
        if ((v.vop == V_IMOD || v.vop == V_IFLOORDIV) && (in.flags & TPLX_F_B_CONST) && in.imm > 0 && (in.imm & (in.imm - 1)) == 0) {
            // constant power-of-two divisor: x % 2^k == x & (2^k - 1), x // 2^k == x >> k under floored semantics; cannot raise
            int k = 0;
            while ((1ll << k) != in.imm) ++k;
            v.in.imm = v.vop == V_IMOD ? in.imm - 1 : k;
            v.vop = v.vop == V_IMOD ? V_IANDK : V_ISHRK;
        }
        pl.ins.push_back(v);
    }
    auto unguarded = [](const VecIns &v) { return v.in.guard == TPLX_NOSLOT; };
    auto reads_slot = [](const VecIns &v, int which) -> int {  // slot read through operand `which` from the register file, or -1
        const uint32_t m = vop_reads(v.vop);
        if (!((m >> which) & 1u)) return -1;
        const uint32_t cf = which == 0 ? TPLX_F_A_CONST : (which == 1 ? TPLX_F_B_CONST : TPLX_F_C_CONST);
        if (v.in.flags & cf) return -1;
        if (which == 0 && (v.xf & VX_A_ACC)) return -1;
        if (which == 1 && (v.xf & VX_B_ACC)) return -1;
        const uint16_t sl = which == 0 ? v.in.a : (which == 1 ? v.in.b : v.in.c);
        return sl == TPLX_NOSLOT ? -1 : (int)sl;
    };
    // is the value instruction i left in slot d read from the slot after position `from` (or an output)?
    auto slot_live_after = [&](size_t from, uint16_t d) {
        for (size_t k = from; k < pl.ins.size(); ++k) {
            const VecIns &v = pl.ins[k];
            for (int w = 0; w < 3; ++w)
                if (reads_slot(v, w) == (int)d) return true;
            if (v.in.guard == d) return true;
            if (vop_has_dst(v.vop) && v.in.dst == d) {
                if (unguarded(v) && !vop_raising(v.vop)) return false;  // fully overwritten (a raising op writes its active rows only)
                return true;                                            // partial write: the old value shows through
            }
        }
        for (const tplx_outcol &oc : outs)
            if (oc.slot == d) return true;
        return false;
    };
    // (a) x % 2^k feeding only the next integer compare
    for (size_t i = 0; i + 1 < pl.ins.size(); ++i) {
        VecIns &m = pl.ins[i], &c = pl.ins[i + 1];
        if (m.vop != V_IANDK || !unguarded(m) || !unguarded(c) || !vop_icmp(c.vop) || (m.in.flags & TPLX_F_A_CONST) || (c.in.flags & TPLX_F_A_CONST)) continue;
        if (c.in.a != m.in.dst || (!(c.in.flags & TPLX_F_B_CONST) && c.in.b == m.in.dst)) continue;
        if (c.in.dst != m.in.dst && slot_live_after(i + 2, m.in.dst)) continue;
        c.in.a = m.in.a;
        c.in.imm2 = m.in.imm;
        c.xf |= VX_A_MASK;
        pl.ins.erase(pl.ins.begin() + (long)i);
    }
    // (b) boolean op feeding only the next FILTER
    for (size_t i = 0; i + 1 < pl.ins.size(); ++i) {
        VecIns &c = pl.ins[i], &f = pl.ins[i + 1];
        if (!vop_pred(c.vop) || f.vop != V_FILTER || !unguarded(c) || !unguarded(f) || (f.in.flags & TPLX_F_A_CONST) || f.in.a != c.in.dst) continue;
        c.xf |= VX_FILTER;
        pl.ins.erase(pl.ins.begin() + (long)i + 1);
    }
    // (c) accumulator operands
    for (size_t i = 0; i + 1 < pl.ins.size(); ++i) {
        const VecIns &pr = pl.ins[i];
        VecIns &co = pl.ins[i + 1];
        if (!unguarded(pr) || !unguarded(co) || !vop_has_dst(pr.vop) || vop_raising(pr.vop) || vop_raising(co.vop) || co.vop == V_RAISE) continue;
        const uint32_t m = vop_reads(co.vop);
        const bool a_is = (m & 1u) && !(co.in.flags & TPLX_F_A_CONST) && co.in.a == pr.in.dst;
        const bool b_is = (m & 2u) && !(co.in.flags & TPLX_F_B_CONST) && co.in.b == pr.in.dst;
        if (a_is) {
            co.xf |= VX_A_ACC;
            if (b_is) co.xf |= VX_B_ACC;  // x op x
        } else if (b_is && co.vop != V_SEL && !(co.xf & VX_A_MASK)) {
            // the accumulator is operand a's home (loading a overwrites it): commute, or flip the comparison, so that the chained
            // value becomes a; ops that are neither (x - acc, x << acc) read the stored slot instead
            uint32_t sw = V_NOP;
            switch (co.vop) {
                case V_IADD: case V_IMUL: case V_IAND: case V_IOR: case V_IXOR: case V_FADD: case V_FMUL: case V_BAND: case V_BOR:
                case V_ICMP_EQ: case V_ICMP_NE: case V_FCMP_EQ: case V_FCMP_NE: sw = co.vop; break;
                case V_ICMP_LT: sw = V_ICMP_GT; break;
                case V_ICMP_GT: sw = V_ICMP_LT; break;
                case V_ICMP_LE: sw = V_ICMP_GE; break;
                case V_ICMP_GE: sw = V_ICMP_LE; break;
                case V_FCMP_LT: sw = V_FCMP_GT; break;
                case V_FCMP_GT: sw = V_FCMP_LT; break;
                case V_FCMP_LE: sw = V_FCMP_GE; break;
                case V_FCMP_GE: sw = V_FCMP_LE; break;
                default: break;
            }
            if (sw != V_NOP) {
                co.vop = sw;
                std::swap(co.in.a, co.in.b);
                std::swap(co.in.imm, co.in.imm2);
                const uint8_t fl = co.in.flags;
                co.in.flags = (uint8_t)((fl & ~(TPLX_F_A_CONST | TPLX_F_B_CONST)) | ((fl & TPLX_F_A_CONST) ? TPLX_F_B_CONST : 0) |
                                        ((fl & TPLX_F_B_CONST) ? TPLX_F_A_CONST : 0));
                co.xf |= VX_A_ACC;
            }
        }
    }
    // (d) results nobody reads from their slot
    for (size_t i = 0; i < pl.ins.size(); ++i) {
        VecIns &v = pl.ins[i];
        if (!unguarded(v) || !vop_has_dst(v.vop) || vop_raising(v.vop) || v.in.dst == TPLX_NOSLOT) continue;
        if (!slot_live_after(i + 1, v.in.dst)) v.xf |= VX_NOSTORE;
    }
    // (e) dense slot numbers for what is still touched
    pl.slot_map.assign(std::max<uint32_t>(n_slots_ir, 1), TPLX_NOSLOT);
    uint32_t next = 0;
    auto touch = [&](uint16_t sl) {
        if (sl != TPLX_NOSLOT && sl < pl.slot_map.size() && pl.slot_map[sl] == TPLX_NOSLOT) pl.slot_map[sl] = (uint16_t)next++;
    };
    for (const VecIns &v : pl.ins) {
        for (int w = 0; w < 3; ++w) {
            const int sl = reads_slot(v, w);
            if (sl >= 0) touch((uint16_t)sl);
        }
        touch(v.in.guard);
        if (vop_has_dst(v.vop) && !(v.xf & VX_NOSTORE)) touch(v.in.dst);
    }
    for (const tplx_outcol &oc : outs) touch(oc.slot);
    pl.n_slots = std::max<uint32_t>(next, 1);
    return pl;
}
// device format of the plan (VInstr, vecvm.cuh) for tiles of T rows: the program sits at the start of shared memory, the register
// file at regs_off with a slot stride of T * 8 bytes
static std::vector<VInstr> vec_encode(const VecPlan &pl, uint32_t T, uint32_t regs_off) {
    std::vector<VInstr> out;
    auto off = [&](uint16_t sl) { return sl == TPLX_NOSLOT || pl.slot_map[sl] == TPLX_NOSLOT ? NOOFF : (uint32_t)pl.slot_map[sl] * T * 8u; };
    for (size_t i = 0; i < pl.ins.size(); ++i) {
        const VecIns &v = pl.ins[i];
        VInstr d{};
        uint32_t xf = v.xf;
        const uint32_t rd = vop_reads(v.vop), self = (uint32_t)(i * sizeof(VInstr));
        if (rd & 1u) {
            if (!(xf & VX_A_ACC)) {
                xf |= VX_LOAD_A;
                if (v.in.flags & TPLX_F_A_CONST) d.pa = self + (uint32_t)offsetof(VInstr, ka);
                else { d.pa = regs_off + off(v.in.a); xf |= VX_A_THREAD; }
            }
        }
        if ((rd & 2u) && !(xf & VX_B_ACC)) {
            if (v.in.flags & TPLX_F_B_CONST) d.pb = self + (uint32_t)offsetof(VInstr, kb);
            else { d.pb = regs_off + off(v.in.b); xf |= VX_B_THREAD; }
        }
        if (rd & 4u) d.pc = off(v.in.c);
        if (vop_has_dst(v.vop)) xf |= VX_RESULT;
        d.op_opidx = v.vop | ((uint32_t)v.in.opidx << 16);
        d.xf = xf;
        d.dst = (v.xf & VX_NOSTORE) ? NOOFF : off(v.in.dst);
        d.guard = off(v.in.guard);
        d.kb[0] = d.kb[1] = (uint64_t)v.in.imm;
        d.ka[0] = d.ka[1] = (uint64_t)v.in.imm2;
        out.push_back(d);
    }
    return out;
}

struct StageDev {
    Device *dev = nullptr;
    DInstr *prog = nullptr;  // pre-decoded program
    DInstr *prog_vec[2] = {nullptr, nullptr};  // the same for the vector kernel (slot stride of T = 1024 / 2048 rows), built on demand
                                               // (written and read under tplx_stage::mu)
    uint8_t *cpool = nullptr;
    int64_t *opids = nullptr;
    HashTable *ht = nullptr;  // HASH endpoint
    std::map<int, jit::Loaded> jit_fn;  // specialised kernels of this stage on this device, by jit::Kind
};

struct tplx_stage {
    tplx_stage_header hdr{};
    std::vector<uint8_t> in_types;    // per input column of the program; "is None" companions appear as TPLX_T_BOOL
    std::vector<int32_t> in_null_of;  // per input column: -1, or the Option[T] column this one is the companion of
    uint32_t n_companions = 0;        // trailing companion columns (the caller's blocks hold in_types.size() - n_companions columns)
    std::vector<tplx_outcol> out_cols;
    std::vector<tplx_acc> accs;
    std::vector<int64_t> opids;
    std::vector<tplx_instr> instrs;
    std::vector<uint8_t> cpool;
    bool has_str = false;
    bool materialises = false;
    uint32_t n_str_out = 0;
    std::vector<StageDev> devs;
    // Run-time state that later blocks are sized from. Blocks of one stage run concurrently on the GPU's execution lanes, so a
    // field may be written by one caller while another reads it: relaxed atomics (any recent value is a valid estimate).
    // adaptive output capacities learnt from earlier blocks (bytes per input row per str out col)
    std::atomic<double> est_bytes_per_row[TPLX_MAX_COLS];
    std::atomic<double> est_exc_per_row{0.0};
    tplx_stage *prefilter = nullptr;  // nested selective stage (row index output), may be null
    std::atomic<bool> prefilter_enabled{true};  // switched off at run time when it turns out not to be selective
    std::atomic<double> est_surv_ratio{-1.0};   // survivors / rows of the last block (prefilter stage): sizes the next block's dense launch
    uint32_t hidden = 0;              // trailing executor-internal output columns
    bool vec_ok = false;              // fixed-width values and vector-VM ops only: eligible for K1v (vecvm.cuh)
    VecPlan vplan;                    // K1v micro-op program (accumulator chains, fused compare/filter), built when vec_ok
    std::vector<tplx_scan_term> scan; // string-scan hint (closed form of a pure filter chain), empty = none
    bool has_fused = false;           // closed-form scan-aggregate hint present and valid
    FusedParams fused{};
    // stage specialiser (jit.inl): live-out slots (the compact register file of the specialised kernels), one binary per kernel kind
    jit::LiveOut jit_live;
    std::map<int, std::shared_ptr<jit::Binary>> jit_bin;
    std::atomic<bool> jit_hot{false};  // a block large enough to pay for the compile has been seen
    std::mutex mu;
};
static constexpr std::memory_order relaxed = std::memory_order_relaxed;

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
// Allocation size of a buffer of `total` string bytes: a 4-byte multiple, readable up to the next 16-byte boundary and 16 bytes
// beyond (the memory contract of strops.cuh: its word-wise readers load every aligned word that holds a byte of a string).
static size_t str_buf_bytes(uint64_t total) { return align_up(total, 16) + 16; }

extern "C" int32_t tplx_gpu_stage_create(const void *desc, uint64_t desc_bytes, tplx_stage **out) {
    if (!desc || !out || desc_bytes < sizeof(tplx_stage_header)) return fail(TPLX_E_BADARG, "stage_create: bad arguments");
    const uint8_t *p = static_cast<const uint8_t *>(desc);
    tplx_stage_header h;
    memcpy(&h, p, sizeof(h));
    if (h.magic != TPLX_IR_MAGIC) return fail(TPLX_E_BADDESC, "stage descriptor: bad magic");
    if (h.version != TPLX_IR_VERSION) return fail(TPLX_E_BADDESC, "stage descriptor: version mismatch");
    if (h.total_bytes != desc_bytes) return fail(TPLX_E_BADDESC, "stage descriptor: size mismatch");
    if (desc_bytes < sizeof(h) + h.prefilter_bytes) return fail(TPLX_E_BADDESC, "stage descriptor: prefilter size");
    if (h.n_in_cols > TPLX_MAX_COLS || h.n_out_cols > TPLX_MAX_COLS || h.n_accs > TPLX_MAX_ACCS || h.n_keys > TPLX_MAX_KEYS)
        return fail(TPLX_E_BADDESC, "stage descriptor: too many columns/accumulators");
    size_t off = sizeof(h);
    auto need = [&](size_t n) { return off + n <= desc_bytes; };
    tplx_stage *s = new tplx_stage();
    s->hdr = h;
    auto bad = [&](const char *m) {
        delete s;
        return fail(TPLX_E_BADDESC, m);
    };
    size_t n = align_up(h.n_in_cols, 8);
    if (!need(n)) return bad("stage descriptor truncated (in_types)");
    s->in_types.assign(p + off, p + off + h.n_in_cols);
    s->in_null_of.assign(h.n_in_cols, -1);
    for (uint32_t c = 0; c < h.n_in_cols; ++c)
        if (s->in_types[c] & TPLX_T_NULLOF) {  // "is None" companion of an Option[T] column: a bool column the executor fills
            s->in_null_of[c] = s->in_types[c] & 0x7F;
            s->in_types[c] = TPLX_T_BOOL;
            ++s->n_companions;
        }
    for (uint32_t c = 0; c < h.n_in_cols; ++c) {
        const bool comp = s->in_null_of[c] >= 0;
        if (comp != (c >= h.n_in_cols - s->n_companions) || (comp && (uint32_t)s->in_null_of[c] >= h.n_in_cols - s->n_companions))
            return bad("stage descriptor: companion columns must follow the physical columns and name one of them");
    }
    off += n;
    n = align_up(h.n_out_cols * sizeof(tplx_outcol), 8);
    if (!need(n)) return bad("stage descriptor truncated (out_cols)");
    s->out_cols.resize(h.n_out_cols);
    memcpy(s->out_cols.data(), p + off, h.n_out_cols * sizeof(tplx_outcol));
    off += n;
    n = h.n_accs * sizeof(tplx_acc);
    if (!need(n)) return bad("stage descriptor truncated (accs)");
    s->accs.resize(h.n_accs);
    memcpy(s->accs.data(), p + off, n);
    off += n;
    n = h.n_ops * sizeof(int64_t);
    if (!need(n)) return bad("stage descriptor truncated (opids)");
    s->opids.resize(h.n_ops);
    memcpy(s->opids.data(), p + off, n);
    off += n;
    n = (size_t)h.n_instr * sizeof(tplx_instr);
    if (!need(n)) return bad("stage descriptor truncated (instrs)");
    s->instrs.resize(h.n_instr);
    memcpy(s->instrs.data(), p + off, n);
    off += n;
    n = align_up(h.const_bytes, 8);
    if (!need(n)) return bad("stage descriptor truncated (const pool)");
    s->cpool.assign(p + off, p + off + h.const_bytes);
    off += n;

    // ---- validate the program (what TransformStage::compile would reject) ----
    const uint32_t ns = h.n_slots;
    auto slot_ok = [&](uint16_t v, uint32_t width) { return v == TPLX_NOSLOT || (uint32_t)v + width <= ns; };
    for (uint32_t i = 0; i < h.n_instr; ++i) {
        const tplx_instr &in = s->instrs[i];
        if (!slot_ok(in.dst, 1) || !slot_ok(in.a, 1) || !slot_ok(in.b, 1) || !slot_ok(in.c, 1) || !slot_ok(in.guard, 1))
            return bad("program: slot out of range");
        if (h.n_ops && in.opidx >= h.n_ops) return bad("program: operator index out of range");
        switch (in.op) {
            case TPLX_OP_LDCOL:
                if (in.imm < 0 || in.imm >= h.n_in_cols) return bad("program: LDCOL column out of range");
                if (in.flags != s->in_types[in.imm]) return bad("program: LDCOL type mismatch");
                break;
            case TPLX_OP_LDS:
                if (((uint64_t)in.imm & 0xFFFFFFFFull) + ((uint64_t)in.imm >> 32) > h.const_bytes)
                    return bad("program: LDS constant out of range");
                break;
            case TPLX_OP_SREPLACE: case TPLX_OP_SCONCAT: case TPLX_OP_SFMTD: case TPLX_OP_I2S:
                s->materialises = true;
                break;
            default: break;
        }
        if (in.op == TPLX_OP_SRFINDK && ((in.flags & TPLX_F_A_CONST) || in.a == TPLX_NOSLOT)) return bad("program: SRFINDK needs a slot operand a");
        if ((in.op >= TPLX_OP_SLEN && in.op <= TPLX_OP_SSTRIP) || in.op == TPLX_OP_S2F || in.op == TPLX_OP_SFINDE || in.op == TPLX_OP_SRFINDK) {
            s->has_str = true;
            // constant string operands are constant-pool views (offset | length << 32)
            auto cs_ok = [&](int64_t enc) { return ((uint64_t)enc & 0xFFFFFFFFull) + ((uint64_t)enc >> 32) <= h.const_bytes; };
            const bool str_b = in.op == TPLX_OP_SFIND || in.op == TPLX_OP_SRFIND || in.op == TPLX_OP_SIN || in.op == TPLX_OP_SEQ || in.op == TPLX_OP_SFINDE || in.op == TPLX_OP_SRFINDK ||
                               in.op == TPLX_OP_SSTARTS || in.op == TPLX_OP_SENDS || in.op == TPLX_OP_SCONCAT || in.op == TPLX_OP_SREPLACE;
            if (in.op != TPLX_OP_SFMTD && in.op != TPLX_OP_I2S && (in.flags & TPLX_F_A_CONST) && !cs_ok(in.imm2)) return bad("program: constant operand a out of range");
            if (str_b && (in.flags & TPLX_F_B_CONST) && !cs_ok(in.imm)) return bad("program: constant operand b out of range");
            if (in.op == TPLX_OP_SREPLACE && (in.flags & TPLX_F_C_CONST) && !cs_ok(in.imm2)) return bad("program: constant operand c out of range");
        }
        if ((in.op == TPLX_OP_SEL || in.op == TPLX_OP_MOV) && (in.flags & 3) == 2) {
            auto cs_ok = [&](int64_t enc) { return ((uint64_t)enc & 0xFFFFFFFFull) + ((uint64_t)enc >> 32) <= h.const_bytes; };
            if ((in.flags & TPLX_F_A_CONST) && !cs_ok(in.imm2)) return bad("program: constant operand a out of range");
            if ((in.flags & TPLX_F_B_CONST) && !cs_ok(in.imm)) return bad("program: constant operand b out of range");
            s->has_str = true;
        }
        if (in.op == TPLX_OP_LDS) s->has_str = true;
    }
    if (h.hidden_out_cols > h.n_out_cols) return bad("stage descriptor: hidden_out_cols out of range");
    uint32_t key_companions = 0;  // HASH: bit k = key column k has its companion
    for (uint32_t k = 0; k < h.n_out_cols; ++k) {
        const tplx_outcol &oc = s->out_cols[k];
        if (!oc.null_of) continue;
        if (h.endpoint == TPLX_EP_HASH) {
            const uint32_t key = oc.null_of - 1u;
            if (oc.type != TPLX_T_BOOL || k < h.n_out_cols - h.hidden_out_cols || k < h.n_keys || key >= h.n_keys ||
                key >= (uint32_t)(h.n_out_cols - h.hidden_out_cols) || (key_companions >> key & 1u))
                return bad("stage descriptor: an `is None` companion of a hash stage must be a hidden bool column of one key column");
            key_companions |= 1u << key;
        } else if (h.endpoint != TPLX_EP_MEMORY || oc.type != TPLX_T_BOOL || k < h.n_out_cols - h.hidden_out_cols ||
                   oc.null_of > h.n_out_cols - h.hidden_out_cols)
            return bad("stage descriptor: an `is None` companion must be a hidden bool column of a visible output column");
    }
    s->hidden = h.hidden_out_cols;
    if (h.prefilter_bytes) {
        if (!need(h.prefilter_bytes) || h.endpoint != TPLX_EP_MEMORY) return bad("stage descriptor: bad prefilter section");
        int32_t prc = tplx_gpu_stage_create(p + off, h.prefilter_bytes, &s->prefilter);
        if (prc) { delete s; return prc; }
        tplx_stage *q = s->prefilter;
        if (q->prefilter || q->hdr.endpoint != TPLX_EP_MEMORY || q->out_cols.size() != 1 || q->out_cols[0].type != TPLX_T_I64 ||
            q->in_types != s->in_types || !s->hidden)
            return bad("stage descriptor: prefilter must be a row-index MEMORY stage over the same input schema");
        off += h.prefilter_bytes;
    }
    if (h.fused_bytes && h.endpoint == TPLX_EP_MEMORY) {
        // string-scan hint: the stage as a list of closed-form filter terms (execution hint; validated here)
        tplx_scan_header sh;
        if (!need(h.fused_bytes) || h.fused_bytes < sizeof(sh)) return bad("stage descriptor: bad scan section");
        memcpy(&sh, p + off, sizeof(sh));
        if (sh.magic != TPLX_SCAN_MAGIC || sh.n_terms == 0 || sh.n_terms > TPLX_MAX_SCAN_TERMS ||
            h.fused_bytes != sizeof(sh) + sh.n_terms * sizeof(tplx_scan_term))
            return bad("stage descriptor: malformed scan section");
        s->scan.resize(sh.n_terms);
        memcpy(s->scan.data(), p + off + sizeof(sh), sh.n_terms * sizeof(tplx_scan_term));
        auto view_ok = [&](uint64_t enc) { return (enc & 0xFFFFFFFFull) + (enc >> 32) <= h.const_bytes; };
        for (const tplx_scan_term &t : s->scan) {
            bool ok = t.col < h.n_in_cols && t.kind <= TPLX_SK_FIXED && t.cmp <= TPLX_CMP_GE && (!h.n_ops || (t.opidx_val < h.n_ops && t.opidx_filter < h.n_ops));
            if (ok && t.kind == TPLX_SK_FIXED) ok = s->in_types[t.col] != TPLX_T_STR;
            if (ok && t.kind != TPLX_SK_FIXED) ok = s->in_types[t.col] == TPLX_T_STR && view_ok(t.needle) && (t.flags & TPLX_SCF_CASE_MASK) <= TPLX_SF_UPPER;
            if (ok && t.kind == TPLX_SK_FIELD_INT) ok = view_ok(t.sep);
            if (!ok) return bad("stage descriptor: scan term references bad columns or constants");
        }
        off += h.fused_bytes;
    } else if (h.fused_bytes) {
        // closed-form scan-aggregate hint (execution hint; validated, and ignored when it does not fit)
        if (!need(h.fused_bytes) || h.fused_bytes < sizeof(tplx_fused_header) || h.endpoint != TPLX_EP_AGGREGATE)
            return bad("stage descriptor: bad fused section");
        tplx_fused_header fh;
        memcpy(&fh, p + off, sizeof(fh));
        if (fh.magic != TPLX_FUSED_MAGIC || fh.n_preds > TPLX_MAX_FUSED_PREDS || fh.n_terms != h.n_accs ||
            h.fused_bytes != sizeof(fh) + fh.n_preds * sizeof(tplx_fused_pred) + fh.n_terms * sizeof(tplx_fused_term))
            return bad("stage descriptor: malformed fused section");
        FusedParams &F = s->fused;
        memset(&F, 0, sizeof(F));
        F.n_preds = fh.n_preds;
        F.n_terms = fh.n_terms;
        memcpy(F.preds, p + off + sizeof(fh), fh.n_preds * sizeof(tplx_fused_pred));
        memcpy(F.terms, p + off + sizeof(fh) + fh.n_preds * sizeof(tplx_fused_pred), fh.n_terms * sizeof(tplx_fused_term));
        bool ok = true;
        auto fixed_col = [&](uint32_t c) { return c < h.n_in_cols && s->in_types[c] != TPLX_T_STR; };
        for (uint32_t i = 0; i < F.n_preds; ++i) ok = ok && fixed_col(F.preds[i].col);
        for (uint32_t i = 0; i < F.n_terms; ++i) {
            const tplx_fused_term &t = F.terms[i];
            ok = ok && t.kind == s->accs[i].kind && t.op <= TPLX_FT_MUL && (t.kind == TPLX_ACC_SUM_I64 || t.kind == TPLX_ACC_SUM_F64);
            if (t.op != TPLX_FT_CONST) ok = ok && fixed_col(t.col_a);
            if (t.op == TPLX_FT_MUL) ok = ok && fixed_col(t.col_b);
        }
        if (!ok) return bad("stage descriptor: fused section references bad columns or accumulators");
        s->has_fused = true;
        off += h.fused_bytes;
    }
    for (auto t : s->in_types) {
        if (t > TPLX_T_STR) return bad("stage descriptor: unknown input type");
        if (t == TPLX_T_STR) s->has_str = true;
    }
    for (auto &oc : s->out_cols) {
        if (oc.type > TPLX_T_STR) return bad("stage descriptor: unknown output type");
        if (!slot_ok(oc.slot, oc.type == TPLX_T_STR ? 2 : 1) || oc.slot == TPLX_NOSLOT) return bad("stage descriptor: output slot out of range");
        if (oc.type == TPLX_T_STR) { s->n_str_out++; s->has_str = true; }
    }
    if (s->n_str_out + 2 > MAX_SCAN) return bad("stage descriptor: too many string output columns");
    for (auto &a : s->accs)
        if (a.kind > TPLX_ACC_MAX_F64 || a.slot >= ns) return bad("stage descriptor: bad accumulator");
    if (h.endpoint > TPLX_EP_HASH) return bad("stage descriptor: unknown endpoint");
    if (h.endpoint == TPLX_EP_AGGREGATE && h.n_accs == 0) return bad("aggregate endpoint without accumulators");
    if (h.endpoint == TPLX_EP_HASH && (h.n_keys == 0 || h.n_keys > h.n_out_cols)) return bad("hash endpoint without key columns");
    for (auto &e : s->est_bytes_per_row) e.store(-1.0, relaxed);
    // K1v eligibility: no string value anywhere and only operations the vector VM implements
    s->vec_ok = !s->has_str && h.endpoint == TPLX_EP_MEMORY && h.n_instr > 0;
    for (const tplx_instr &in : s->instrs) {
        switch (in.op) {
            case TPLX_OP_LDCOL: case TPLX_OP_LDI: case TPLX_OP_LDROW: case TPLX_OP_MOV: case TPLX_OP_SEL: case TPLX_OP_IADD: case TPLX_OP_ISUB:
            case TPLX_OP_IMUL: case TPLX_OP_IFLOORDIV: case TPLX_OP_IMOD: case TPLX_OP_INEG: case TPLX_OP_IAND: case TPLX_OP_IOR: case TPLX_OP_IXOR:
            case TPLX_OP_ISHL: case TPLX_OP_ISHR: case TPLX_OP_IABS: case TPLX_OP_FADD: case TPLX_OP_FSUB: case TPLX_OP_FMUL: case TPLX_OP_FDIV:
            case TPLX_OP_FMOD: case TPLX_OP_FNEG: case TPLX_OP_FFLOORDIV: case TPLX_OP_FABS: case TPLX_OP_I2F: case TPLX_OP_F2I: case TPLX_OP_ICMP:
            case TPLX_OP_FCMP: case TPLX_OP_BAND: case TPLX_OP_BOR: case TPLX_OP_BNOT: case TPLX_OP_FILTER: case TPLX_OP_RAISE: case TPLX_OP_NOP:
                break;
            default: s->vec_ok = false;
        }
        if ((in.op == TPLX_OP_SEL || in.op == TPLX_OP_MOV) && (in.flags & 3) != 1) s->vec_ok = false;
    }
    if (s->vec_ok) s->vplan = vec_plan(s->instrs, s->out_cols, h.n_slots);
    s->jit_live = jit::liveout(s->out_cols, s->accs, h.n_slots);
    *out = s;
    return TPLX_OK;
}

// tplx_instr -> device format: slot numbers become byte offsets into a thread's register column
// (the vector kernel has its own planner: vec_plan / vec_encode)
static std::vector<DInstr> predecode(const std::vector<tplx_instr> &ins, uint32_t slot_bytes = NT * 8) {
    std::vector<DInstr> out(ins.size());
    auto off = [slot_bytes](uint16_t slot) { return slot == TPLX_NOSLOT ? NOOFF : (uint32_t)slot * slot_bytes; };
    for (size_t i = 0; i < ins.size(); ++i) {
        const tplx_instr &in = ins[i];
        DInstr d{};
        d.op_flags = (uint32_t)in.op | ((uint32_t)in.flags << 8) | ((uint32_t)in.opidx << 16);
        d.dst = off(in.dst);
        d.a = off(in.a);
        d.b = off(in.b);
        d.c = off(in.c);
        d.guard = off(in.guard);
        d.imm = in.imm;
        d.imm2 = in.imm2;
        out[i] = d;
    }
    return out;
}

// ---- stage specialiser: compile (once per stage and kernel kind) and load (once per device) -------------------------------------
static void jit_compile_job(std::shared_ptr<jit::Binary> bin, std::string src, int kind, int minb, size_t n_instr) {
    jit::compile(*bin, src, kind, minb);
    if (getenv("TPLX_TRACE") || (bin->failed && getenv("TPLX_JIT_VERBOSE")))
        fprintf(stderr, "[tplx] specialiser: kind %d, %zu instructions -> %zu B cubin in %.0f ms%s%s\n", kind, n_instr, bin->cubin.size(), bin->compile_ms,
                bin->failed ? " FAILED: " : "", bin->failed ? bin->log.c_str() : "");
    if (const char *dir = getenv("TPLX_JIT_DUMP")) {  // evidence / debugging: the generated row function and the cubin
        const std::string base = std::string(dir) + "/tplx_jit_k" + std::to_string(kind) + "_" + std::to_string(n_instr) + "ins";
        if (FILE *f = fopen((base + ".cuh").c_str(), "w")) { fwrite(bin->source.data(), 1, bin->source.size(), f); fclose(f); }
        if (!bin->failed)
            if (FILE *f = fopen((base + ".cubin").c_str(), "wb")) { fwrite(bin->cubin.data(), 1, bin->cubin.size(), f); fclose(f); }
    }
    bin->ready.store(1, std::memory_order_release);
}
// wait = false: the compile runs on a background thread and the returned binary may not be ready yet (ready == 0)
static std::shared_ptr<jit::Binary> jit_binary(tplx_stage *s, int kind, int minb, bool wait) {  // s->mu held
    auto it = s->jit_bin.find(kind);
    if (it != s->jit_bin.end()) {
        if (wait && !it->second->ready.load(std::memory_order_acquire) && it->second->worker.joinable()) it->second->worker.join();
        return it->second;
    }
    auto bin = std::make_shared<jit::Binary>();
    s->jit_bin[kind] = bin;
    std::string src = jit::generate(s->hdr, s->instrs, s->in_types, s->jit_live, s->out_cols, kind);
    if (wait) jit_compile_job(bin, std::move(src), kind, minb, s->instrs.size());
    else bin->worker = std::thread(jit_compile_job, bin, std::move(src), kind, minb, s->instrs.size());
    return bin;
}
// resident CTAs per SM the specialised kernel's register allocation must allow
static int jit_minb(const tplx_stage *s, int kind) {
    switch (kind) {
        case jit::K_VEC4: return 8;
        case jit::K_WIDE4: return 3;
        case jit::K_RE2: return 6;
        case jit::K_VEC2: return 3;
        case jit::K_MASK: return 4;
        default: return 3;
    }
}
static bool jit_wanted(tplx_stage *s, uint64_t block_rows) {
    const int m = jit::mode();
    if (m <= 0 || s->instrs.empty()) return false;
    if (m >= 2 || block_rows >= jit::min_rows()) s->jit_hot.store(true, relaxed);
    return s->jit_hot.load(relaxed);
}
// nullptr: not available (NVRTC / driver entry points missing, compile or load failed) — the interpreting kernel runs instead
static jit::Loaded *jit_get(tplx_stage *s, StageDev *sd, int kind, int minb) {
    std::lock_guard<std::mutex> lk(s->mu);
    auto it = sd->jit_fn.find(kind);
    if (it != sd->jit_fn.end()) return it->second.failed ? nullptr : &it->second;
    jit::Loaded ld;
    jit::CuDrv *cu = jit::cudrv_api();
    std::shared_ptr<jit::Binary> bin = jit_binary(s, kind, minb, jit::synchronous());
    if (!bin->ready.load(std::memory_order_acquire)) return nullptr;  // still compiling: this block runs on the interpreting kernel
    if (!cu || bin->failed) ld.failed = true;
    if (!ld.failed) {
        cudaSetDevice(sd->dev->id);
        cudaFree(0);  // the runtime's primary context is current on this thread
        int rc = cu->ModuleLoadData(&ld.mod, bin->cubin.data());
        if (!rc) rc = cu->ModuleGetFunction(&ld.fn, ld.mod, "tplx_jit_kernel");
        if (!rc) rc = cu->FuncSetAttribute(ld.fn, jit::CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, sd->dev->smem_optin);
        if (!rc) cu->FuncGetAttribute(&ld.regs, jit::CU_FUNC_ATTRIBUTE_NUM_REGS, ld.fn);
        if (rc) {
            const char *msg = nullptr;
            cu->GetErrorString(rc, &msg);
            if (getenv("TPLX_TRACE") || getenv("TPLX_JIT_VERBOSE")) fprintf(stderr, "[tplx] specialiser: loading kind %d failed: %s\n", kind, msg ? msg : "?");
            ld.failed = true;
        } else if (getenv("TPLX_TRACE"))
            fprintf(stderr, "[tplx] specialiser: kind %d loaded on device %d, %d registers/thread\n", kind, sd->dev->id, ld.regs);
    }
    auto &slot = sd->jit_fn[kind];
    slot = ld;
    return slot.failed ? nullptr : &slot;
}
static bool jit_pending(tplx_stage *s, int kind) {  // a background compile of this kind is still running
    std::lock_guard<std::mutex> lk(s->mu);
    auto it = s->jit_bin.find(kind);
    return it != s->jit_bin.end() && !it->second->ready.load(std::memory_order_acquire);
}
static int32_t jit_launch(jit::Loaded *jf, uint32_t grid, uint32_t smem, cudaStream_t st, const void *params) {
    void *args[] = {const_cast<void *>(params)};
    const int rc = jit::cudrv_api()->LaunchKernel(jf->fn, grid, 1, 1, NT, 1, 1, smem, (void *)st, args, nullptr);
    if (rc) {
        const char *msg = nullptr;
        jit::cudrv_api()->GetErrorString(rc, &msg);
        return fail(TPLX_E_CUDA, std::string("specialised kernel launch: ") + (msg ? msg : "?"));
    }
    return TPLX_OK;
}
static int jit_occupancy(jit::Loaded *jf, uint32_t smem) {
    int occ = 0;
    if (jit::cudrv_api()->OccupancyMaxActiveBlocksPerMultiprocessor(&occ, jf->fn, NT, smem)) occ = 0;
    return occ;
}

static int32_t stage_dev(tplx_stage *s, Device *d, StageDev **out) {
    std::lock_guard<std::mutex> lk(s->mu);
    for (auto &sd : s->devs)
        if (sd.dev->id == d->id) { *out = &sd; return TPLX_OK; }  // lanes of one GPU share the device copies
    s->devs.reserve(16);
    StageDev sd;
    sd.dev = d;
    CU(cudaSetDevice(d->id));
    std::vector<DInstr> dec = predecode(s->instrs);
    size_t nb = std::max<size_t>(dec.size() * sizeof(DInstr), 16);
    CU(cudaMalloc(&sd.prog, nb));
    CU(cudaMemcpy(sd.prog, dec.data(), dec.size() * sizeof(DInstr), cudaMemcpyHostToDevice));
    CU(cudaMalloc(&sd.cpool, str_buf_bytes(s->cpool.size())));
    CU(cudaMemcpy(sd.cpool, s->cpool.data(), s->cpool.size(), cudaMemcpyHostToDevice));
    CU(cudaMalloc(&sd.opids, std::max<size_t>(s->opids.size() * 8, 16)));
    CU(cudaMemcpy(sd.opids, s->opids.data(), s->opids.size() * 8, cudaMemcpyHostToDevice));
    s->devs.push_back(sd);
    *out = &s->devs.back();
    return TPLX_OK;
}

extern "C" int32_t tplx_gpu_stage_vec_plan(const tplx_stage *s, tplx_vec_uop *out, uint32_t cap, uint32_t *n_uops, uint32_t *n_slots,
                                           uint16_t *out_slots, uint32_t cap_out) {
    if (!s || !n_uops) return fail(TPLX_E_BADARG, "stage_vec_plan: bad arguments");
    *n_uops = s->vec_ok ? (uint32_t)s->vplan.ins.size() : 0;
    if (n_slots) *n_slots = s->vec_ok ? s->vplan.n_slots : 0;
    if (!s->vec_ok) return TPLX_OK;
    const VecPlan &pl = s->vplan;
    auto dense = [&](uint16_t sl) { return sl == TPLX_NOSLOT || sl >= pl.slot_map.size() ? (uint16_t)TPLX_NOSLOT : pl.slot_map[sl]; };
    for (uint32_t i = 0; out && i < cap && i < pl.ins.size(); ++i) {
        const VecIns &v = pl.ins[i];
        tplx_vec_uop u{};
        u.vop = v.vop;
        u.xflags = v.xf;
        u.flags = v.in.flags;
        u.opidx = v.in.opidx;
        u.dst = (v.xf & VX_NOSTORE) ? (uint16_t)TPLX_NOSLOT : dense(v.in.dst);
        u.a = dense(v.in.a);
        u.b = dense(v.in.b);
        u.c = dense(v.in.c);
        u.guard = dense(v.in.guard);
        u.imm = v.in.imm;
        u.imm2 = v.in.imm2;
        out[i] = u;
    }
    for (uint32_t c = 0; out_slots && c < cap_out && c < s->out_cols.size(); ++c) out_slots[c] = dense(s->out_cols[c].slot);
    return TPLX_OK;
}

extern "C" int32_t tplx_gpu_stage_specialise(tplx_stage *s, int32_t kind, int32_t compile, char *src, uint64_t src_cap, uint64_t *src_len,
                                             uint64_t *cubin_bytes, char *log, uint64_t log_cap) {
    if (!s || !jit::is_kind(kind)) return fail(TPLX_E_BADARG, "stage_specialise: bad arguments");
    if (jit::is_fixed_width(kind) && !s->vec_ok) return fail(TPLX_E_UNSUPPORTED, "stage_specialise: not a fixed-width MEMORY stage");
    std::string text;
    size_t nb = 0;
    std::string lg;
    if (compile) {
        std::lock_guard<std::mutex> lk(s->mu);
        std::shared_ptr<jit::Binary> bin = jit_binary(s, kind, jit_minb(s, kind), true);
        text = bin->source;
        nb = bin->failed ? 0 : bin->cubin.size();
        lg = bin->log;
    } else text = jit::generate(s->hdr, s->instrs, s->in_types, s->jit_live, s->out_cols, kind);
    if (src_len) *src_len = text.size();
    if (src && src_cap) {
        const size_t n = std::min<size_t>(text.size(), src_cap - 1);
        memcpy(src, text.data(), n);
        src[n] = 0;
    }
    if (cubin_bytes) *cubin_bytes = nb;
    if (log && log_cap) {
        const size_t n = std::min<size_t>(lg.size(), log_cap - 1);
        memcpy(log, lg.data(), n);
        log[n] = 0;
    }
    return TPLX_OK;
}

extern "C" int32_t tplx_gpu_stage_destroy(tplx_stage *s) {
    if (!s) return TPLX_OK;
    for (auto &sd : s->devs) {
        cudaSetDevice(sd.dev->id);
        cudaStreamSynchronize(sd.dev->stream);
        cudaFree(sd.prog);
        cudaFree(sd.prog_vec[0]);
        cudaFree(sd.prog_vec[1]);
        cudaFree(sd.cpool);
        cudaFree(sd.opids);
        if (sd.ht) hash_table_destroy(sd.ht);
        for (auto &kv : sd.jit_fn)
            if (kv.second.mod) jit::cudrv_api()->ModuleUnload(kv.second.mod);
    }
    if (s->prefilter) tplx_gpu_stage_destroy(s->prefilter);
    for (auto &kv : s->jit_bin)
        if (kv.second->worker.joinable()) kv.second->worker.join();
    delete s;
    return TPLX_OK;
}

// ---------------------------------------------------------------------------------------------
// blocks
// ---------------------------------------------------------------------------------------------
struct tplx_block {
    Device *dev = nullptr;
    uint64_t n_rows = 0;
    std::vector<ColIn> cols;           // device pointers
    std::vector<uint64_t> data_bytes;  // per column
    std::vector<void *> owned;         // allocations to free
    cudaEvent_t ready = nullptr;       // recorded on the copy stream when the upload has been enqueued
    std::vector<uint8_t> mapped;       // per column: 1 = read in place from page-locked host memory (run_host);
                                       // 2 = lazy CSV column: data = CSV text, offsets = (uint64) cell references (K6)
    uint8_t csv_quote = '"';
    std::vector<const uint32_t *> valid;  // per column: validity bitmap of an Option[T] column (bit r & 31 of word r >> 5 set = present), or nullptr
};

extern "C" int32_t tplx_gpu_block_upload(int32_t device, const tplx_column *cols, uint32_t n_cols, uint64_t n_rows,
                                         tplx_block **out) {
    Device *d = get_device(device);
    if (!d) return fail(TPLX_E_NODEVICE, "block_upload: device not initialised (no CPU fallback)");
    if (!cols || !out || n_cols > TPLX_MAX_COLS) return fail(TPLX_E_BADARG, "block_upload: bad arguments");
    CU(cudaSetDevice(d->id));
    tplx_block *b = new tplx_block();
    b->dev = d;
    b->n_rows = n_rows;
    for (uint32_t c = 0; c < n_cols; ++c) {
        ColIn ci{};
        ci.type = cols[c].type;
        uint64_t nb = cols[c].type == TPLX_T_STR ? cols[c].data_bytes : n_rows * 8;
        void *dd = nullptr;
        CU(cudaMallocAsync(&dd, str_buf_bytes(nb), d->copy_stream));
        b->owned.push_back(dd);
        if (nb) CU(cudaMemcpyAsync(dd, cols[c].data, nb, cudaMemcpyHostToDevice, d->copy_stream));
        ci.data = dd;
        if (cols[c].type == TPLX_T_STR) {
            void *od = nullptr;
            CU(cudaMallocAsync(&od, (n_rows + 1) * 4, d->copy_stream));
            b->owned.push_back(od);
            CU(cudaMemcpyAsync(od, cols[c].offsets, (n_rows + 1) * 4, cudaMemcpyHostToDevice, d->copy_stream));
            ci.offsets = static_cast<const uint32_t *>(od);
        }
        b->cols.push_back(ci);
        b->data_bytes.push_back(nb);
        const uint32_t *vd = nullptr;
        if (cols[c].valid) {  // Option[T] column (Serializer.cc:1041-1059 keeps the same information as a per-row bitmap)
            void *vp = nullptr;
            const size_t vb = (n_rows + 31) / 32 * 4;
            CU(cudaMallocAsync(&vp, vb + 16, d->copy_stream));
            b->owned.push_back(vp);
            if (vb) CU(cudaMemcpyAsync(vp, cols[c].valid, vb, cudaMemcpyHostToDevice, d->copy_stream));
            vd = static_cast<const uint32_t *>(vp);
        }
        b->valid.push_back(vd);
    }
    CU(cudaEventCreateWithFlags(&b->ready, cudaEventDisableTiming));
    CU(cudaEventRecord(b->ready, d->copy_stream));
    *out = b;
    return TPLX_OK;
}

extern "C" int32_t tplx_gpu_block_wrap_device(int32_t device, const tplx_column *cols, uint32_t n_cols,
                                              uint64_t n_rows, tplx_block **out) {
    Device *d = get_device(device);
    if (!d) return fail(TPLX_E_NODEVICE, "block_wrap_device: device not initialised");
    if (!cols || !out || n_cols > TPLX_MAX_COLS) return fail(TPLX_E_BADARG, "block_wrap_device: bad arguments");
    tplx_block *b = new tplx_block();
    b->dev = d;
    b->n_rows = n_rows;
    for (uint32_t c = 0; c < n_cols; ++c) {
        ColIn ci{};
        ci.type = cols[c].type;
        ci.data = cols[c].data;
        ci.offsets = cols[c].offsets;
        b->cols.push_back(ci);
        b->data_bytes.push_back(cols[c].type == TPLX_T_STR ? cols[c].data_bytes : n_rows * 8);
        b->valid.push_back(cols[c].valid);
    }
    *out = b;
    return TPLX_OK;
}

extern "C" int32_t tplx_gpu_block_rows(const tplx_block *b, uint64_t *n_rows) {
    if (!b || !n_rows) return fail(TPLX_E_BADARG, "block_rows: bad arguments");
    *n_rows = b->n_rows;
    return TPLX_OK;
}

extern "C" int32_t tplx_gpu_block_column_bytes(const tplx_block *b, uint64_t *bytes, uint32_t max_cols, uint32_t *n_cols) {
    if (!b || !n_cols || (!bytes && max_cols)) return fail(TPLX_E_BADARG, "block_column_bytes: bad arguments");
    *n_cols = (uint32_t)b->cols.size();
    for (uint32_t c = 0; c < b->cols.size() && c < max_cols; ++c)
        bytes[c] = b->data_bytes[c] + (b->cols[c].type == TPLX_T_STR ? (b->n_rows + 1) * 4 : 0);
    return TPLX_OK;
}

extern "C" int32_t tplx_gpu_block_fetch_validity(const tplx_block *b, uint32_t col, uint32_t *words, uint32_t *nullable) {
    if (!b || !nullable || col >= b->cols.size()) return fail(TPLX_E_BADARG, "block_fetch_validity: bad arguments");
    const uint32_t *v = col < b->valid.size() ? b->valid[col] : nullptr;
    *nullable = v ? 1u : 0u;
    const uint64_t n_words = (b->n_rows + 31) / 32;
    if (!v || !words || !n_words) return TPLX_OK;
    CU(cudaSetDevice(b->dev->id));
    if (b->ready) CU(cudaEventSynchronize(b->ready));
    CU(cudaMemcpy(words, v, n_words * 4, cudaMemcpyDeviceToHost));
    return TPLX_OK;
}

extern "C" int32_t tplx_gpu_block_free(tplx_block *b) {
    if (!b) return TPLX_OK;
    cudaSetDevice(b->dev->id);
    for (void *p : b->owned) cudaFreeAsync(p, b->dev->stream);
    if (b->ready) cudaEventDestroy(b->ready);
    delete b;
    return TPLX_OK;
}

// ---------------------------------------------------------------------------------------------
// results
// ---------------------------------------------------------------------------------------------
struct tplx_result {
    Device *dev = nullptr;
    tplx_stage *stage = nullptr;
    const tplx_block *block = nullptr;  // borrowed, needed for exception row gather
    uint64_t n_in = 0, n_out = 0, n_exc = 0;
    std::vector<OutCol> out;
    std::vector<uint8_t> out_types;
    std::vector<uint64_t> str_bytes;
    std::vector<uint32_t *> out_valid;  // per output column: validity bitmap of a nullable column, or nullptr (may be shorter than out)
    tplx_exception_rec *exc = nullptr;
    uint64_t *agg_out = nullptr;
    uint32_t n_accs = 0;
    std::vector<void *> owned;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, evk0 = nullptr, evk1 = nullptr;
    double kernel_ms = 0, total_ms = 0, kernel_ms_extra = 0;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> extra_ev;  // further kernel intervals on the lane's stream (timed lazily in result_info)
    uint32_t hidden = 0;  // trailing internal output columns
    uint64_t h2d_bytes = 0;       // explicit host->device copies of inputs (run_host)
    uint32_t zero_copy_cols = 0;  // input columns read in place from page-locked host memory
    uint32_t launches = 0;
    uint32_t jit_launches = 0;  // of those: kernels produced by the stage specialiser
    uint32_t lane = 0;          // execution lane that ran the block (0 = the device's primary lane, 1 = its `alt`)
    bool owns_block = false;
    tplx_block *owned_block = nullptr;
    tplx_block *expanded_block = nullptr;  // the input block plus the `is None` companions of its Option[T] columns (tplx_gpu_stage_run)
    // mask stage temporaries (run_mask), needed when the exception records have to be expanded again with the exact capacity
    uint32_t *mask_keep = nullptr, *mask_exc = nullptr, *mask_codes = nullptr, mask_words = 0;
    uint64_t *mask_part = nullptr;
};

extern "C" int32_t tplx_gpu_result_free(tplx_result *r) {
    if (!r) return TPLX_OK;
    cudaSetDevice(r->dev->id);
    for (void *p : r->owned) cudaFreeAsync(p, r->dev->stream);
    if (r->ev0) cudaEventDestroy(r->ev0);
    if (r->ev1) cudaEventDestroy(r->ev1);
    if (r->evk0) cudaEventDestroy(r->evk0);
    if (r->evk1) cudaEventDestroy(r->evk1);
    for (auto &e : r->extra_ev) { cudaEventDestroy(e.first); cudaEventDestroy(e.second); }
    if (r->expanded_block) tplx_gpu_block_free(r->expanded_block);
    if (r->owned_block) tplx_gpu_block_free(r->owned_block);
    delete r;
    return TPLX_OK;
}

// shared-memory layout; must mirror stage_rows_kernel / stage_agg_kernel
struct Layout {
    uint32_t cols_off, regs_off, stage_off, misc_off, total;
    uint32_t stash_off = 0;
    bool inplace = false;
    std::vector<uint32_t> col_stage_off;
};
// inplace (rows endpoint, R == 1): no staging area, the write phase reads the outputs from the register file
// jit: layout of the specialised kernel — no program in shared memory, the register file holds the live-out slots only
static Layout make_layout(const tplx_stage *s, uint32_t R, bool rows_ep, bool inplace = false, bool jit = false) {
    Layout L;
    L.inplace = inplace && rows_ep && R == 1;
    const uint32_t T = R * NT, W = T / 32;
    size_t off = jit ? 16 : align_up(std::max<size_t>(s->instrs.size(), 1) * sizeof(DInstr), 16);
    L.cols_off = (uint32_t)off;
    off = align_up(off + std::max<size_t>(s->in_types.size(), 1) * sizeof(ColIn), 16);
    L.regs_off = (uint32_t)off;
    uint32_t nslots = std::max<uint32_t>(std::max<uint32_t>(jit ? (uint32_t)s->jit_live.slots.size() : s->hdr.n_slots, s->n_str_out), 1);
    off = align_up(off + (size_t)nslots * NT * 8, 16);
    L.stage_off = (uint32_t)off;
    if (rows_ep) {
        size_t so = 0;
        for (auto &oc : s->out_cols) {
            L.col_stage_off.push_back((uint32_t)so);
            if (!L.inplace) so += (size_t)T * (oc.type == TPLX_T_STR ? 16 : 8);
        }
        off = align_up(off + so, 16);
        L.misc_off = (uint32_t)off;
        // bitmaps + word prefixes, codes of raising rows (in place: kept in slot 0 of the row), scan values, ticket
        off += (size_t)(4 * W + 2 + (L.inplace ? 0 : T)) * 4 + (size_t)(2 * MAX_SCAN) * 8 + 16;
        off = align_up(off, 16);
        L.stash_off = (uint32_t)off;
        off += (size_t)s->n_str_out * (NT / 32) * 4;
    } else {
        L.misc_off = (uint32_t)off;
        off += (size_t)(NT / 32) * std::max<size_t>(s->accs.size(), 1) * 8;
    }
    L.total = (uint32_t)align_up(off, 16);
    return L;
}
// shared-memory layout of the fixed-width kernels (vecvm.cuh) with T-row tiles: program (16 bytes in a specialised kernel) | cols |
// register file (output columns are staged in place: a slot is indexed by the local row) | misc: 32 group counts per 2048-row
// sub-batch, K1v's exception codes (exc_codes: one word per row of the tile), look-back scratch, ticket
static Layout vec_layout(const tplx_stage *s, size_t prog_bytes, uint32_t T, size_t regs_bytes, bool exc_codes) {
    Layout L;
    L.cols_off = (uint32_t)align_up(prog_bytes, 16);
    L.regs_off = L.stage_off = (uint32_t)align_up(L.cols_off + std::max<size_t>(s->in_types.size(), 1) * sizeof(ColIn), 16);
    L.misc_off = (uint32_t)align_up(L.regs_off + regs_bytes, 16);
    const size_t misc = (size_t)std::max<uint32_t>(T / 2048, 1) * 32 * 4 + (exc_codes ? (size_t)T * 4 : 0) + (size_t)(4 * (NT / 32)) * 8 + 16;
    L.total = (uint32_t)align_up(L.misc_off + misc, 16);
    return L;
}

static int32_t ensure_scratch(Device *d, size_t bytes) {
    if (bytes <= d->scratch_bytes) return TPLX_OK;
    CU(cudaStreamSynchronize(d->stream));
    if (d->scratch) CU(cudaFree(d->scratch));
    d->scratch = nullptr;
    d->scratch_bytes = 0;
    CU(cudaMalloc(&d->scratch, bytes));
    d->scratch_bytes = bytes;
    return TPLX_OK;
}

static int32_t run_rows(tplx_stage *s, StageDev *sd, const tplx_block *b, int64_t first_row_no, tplx_result *r,
                        const uint64_t *rowlist, uint64_t n_list, const std::vector<ColIn> *cols_override = nullptr,
                        const uint64_t *n_work_dev = nullptr);
constexpr int32_t TPLX_INTERNAL_RETRY = 1;  // run_rows with n_work_dev: the device-side count exceeded the estimated capacity
static int32_t device_scan(Device *d, const uint64_t *in, uint64_t *out, uint64_t n, bool write_total);
static int32_t device_scan_batched(Device *d, uint64_t *arrays, uint64_t stride, uint32_t K, uint64_t n);
static int32_t run_rows_prefiltered(tplx_stage *s, StageDev *sd, const tplx_block *b, int64_t first_row_no, tplx_result *r);
static int32_t run_mask(tplx_stage *ps, StageDev *psd, const tplx_block *b, tplx_result *ra, bool no_wait, uint64_t **totals_dev, uint64_t *cap_exc_out);
static int32_t run_agg(tplx_stage *s, StageDev *sd, const tplx_block *b, tplx_result *r);
static int32_t run_hash(tplx_stage *s, StageDev *sd, const tplx_block *b, tplx_result *r);

static int32_t stage_run_impl(tplx_stage *s, const tplx_block *b, int64_t first_row_no, tplx_result **out);
template <typename T>
static int32_t dalloc(tplx_result *r, T **p, size_t count);

// The block plus one "is None" companion column (TPLX_T_BOOL) per entry of `of`: 1 where column of[j] holds None, expanded from that
// column's validity bitmap (all zeros where the column has no bitmap: it holds no None). The companions are filled on the copy
// stream; the new block's `ready` event covers them.
static int32_t expand_companions(const tplx_block *b, const std::vector<uint32_t> &of, tplx_block **out) {
    for (uint8_t m : b->mapped)
        if (m) return fail(TPLX_E_UNSUPPORTED, "stage_run: a stage with Option[T] inputs needs device-resident block columns");
    Device *d = b->dev;
    CU(cudaSetDevice(d->id));
    tplx_block *x = new tplx_block();
    x->dev = d;
    x->n_rows = b->n_rows;
    x->cols = b->cols;
    x->data_bytes = b->data_bytes;
    x->valid = b->valid;
    x->valid.resize(b->cols.size(), nullptr);
    x->csv_quote = b->csv_quote;
    if (b->ready) CU(cudaStreamWaitEvent(d->copy_stream, b->ready, 0));
    const uint64_t n = b->n_rows;
    for (const uint32_t c : of) {
        void *buf = nullptr;
        CU(cudaMallocAsync(&buf, n * 8 + 16, d->copy_stream));
        x->owned.push_back(buf);
        const uint32_t *v = c < b->valid.size() ? b->valid[c] : nullptr;
        if (v && n) valid_expand_kernel<<<(uint32_t)((n + 255) / 256), 256, 0, d->copy_stream>>>(v, n, static_cast<uint64_t *>(buf));
        else CU(cudaMemsetAsync(buf, 0, n * 8 + 16, d->copy_stream));  // a column without a bitmap holds no None
        ColIn ci{};
        ci.type = TPLX_T_BOOL;
        ci.data = buf;
        x->cols.push_back(ci);
        x->data_bytes.push_back(n * 8);
        x->valid.push_back(nullptr);
    }
    CU(cudaGetLastError());
    CU(cudaEventCreateWithFlags(&x->ready, cudaEventDisableTiming));
    CU(cudaEventRecord(x->ready, d->copy_stream));
    *out = x;
    return TPLX_OK;
}

// Option[T] columns on the way in and out of a stage (option.cuh): companions of the input columns are expanded from the block's
// validity bitmaps, companions of the output columns are packed into the result's validity bitmaps.
extern "C" int32_t tplx_gpu_stage_run(tplx_stage *s, const tplx_block *b, int64_t first_row_no, tplx_result **out) {
    if (!s || !b || !out) return fail(TPLX_E_BADARG, "stage_run: bad arguments");
    tplx_block *x = nullptr;
    if (s->n_companions && b->cols.size() + s->n_companions == s->in_types.size()) {
        const std::vector<uint32_t> of(s->in_null_of.begin() + b->cols.size(), s->in_null_of.end());
        int32_t rc = expand_companions(b, of, &x);
        if (rc) return rc;
    }
    int32_t rc = stage_run_impl(s, x ? x : b, first_row_no, out);
    if (rc) {
        if (x) tplx_gpu_block_free(x);
        return rc;
    }
    tplx_result *r = *out;
    if (x) r->expanded_block = x;  // the expanded block lives as long as the result (exception rows are gathered from it)
    bool any = false;
    for (const tplx_outcol &oc : s->out_cols) any = any || oc.null_of;
    if (any && s->hdr.endpoint == TPLX_EP_MEMORY) {
        Device *d = r->dev;
        CU(cudaSetDevice(d->id));
        r->out_valid.assign(r->out.size(), nullptr);
        for (size_t k = 0; k < s->out_cols.size() && k < r->out.size(); ++k) {
            if (!s->out_cols[k].null_of) continue;
            uint32_t *w = nullptr;
            int32_t rc2 = dalloc(r, &w, (r->n_out + 31) / 32 + 1);
            if (rc2) return rc2;
            if (r->n_out) valid_pack_kernel<<<(uint32_t)((r->n_out + 255) / 256), 256, 0, d->stream>>>(r->out[k].data, r->n_out, w);
            r->out_valid[s->out_cols[k].null_of - 1] = w;
            r->launches += 1;
        }
        CU(cudaGetLastError());
        CU(cudaEventRecord(r->ev1, d->stream));
        CU(cudaStreamSynchronize(d->stream));
    }
    return TPLX_OK;
}

static int32_t stage_run_impl(tplx_stage *s, const tplx_block *b, int64_t first_row_no, tplx_result **out) {
    if (!s || !b || !out) return fail(TPLX_E_BADARG, "stage_run: bad arguments");
    if (b->cols.size() != s->in_types.size()) return fail(TPLX_E_BADARG, "stage_run: block column count != stage input schema");
    for (size_t c = 0; c < b->cols.size(); ++c)
        if ((uint8_t)b->cols[c].type != s->in_types[c]) return fail(TPLX_E_BADARG, "stage_run: block column type != stage input schema");
    Device *d = b->dev;
    // several execution lanes per GPU: a concurrent caller does not wait for the first one's kernels, it takes the next
    // free lane (hash stages keep to the primary lane: one table per device)
    std::unique_lock<std::mutex> lk(d->mu, std::try_to_lock);
    uint32_t lane = 0;
    while (!lk.owns_lock()) {
        if (s->hdr.endpoint != TPLX_EP_HASH && d->alt) {
            d = d->alt;
            ++lane;
            lk = d->alt ? std::unique_lock<std::mutex>(d->mu, std::try_to_lock) : std::unique_lock<std::mutex>(d->mu);
        } else {
            lk = std::unique_lock<std::mutex>(d->mu);
        }
    }
    CU(cudaSetDevice(d->id));
    StageDev *sd = nullptr;
    int32_t rc = stage_dev(s, b->dev, &sd);
    if (rc) return rc;
    tplx_result *r = new tplx_result();
    r->dev = d;
    r->lane = lane;
    r->stage = s;
    r->block = b;
    r->n_in = b->n_rows;
    CU(cudaEventCreate(&r->ev0));
    CU(cudaEventCreate(&r->ev1));
    CU(cudaEventCreate(&r->evk0));
    CU(cudaEventCreate(&r->evk1));
    if (b->ready) CU(cudaStreamWaitEvent(d->stream, b->ready, 0));
    CU(cudaEventRecord(r->ev0, d->stream));
    switch (s->hdr.endpoint) {
        case TPLX_EP_MEMORY: {
            bool lazy = false;
            for (uint8_t m : b->mapped) lazy = lazy || m == 2;
            // lazy columns are materialised between the two launches, so such blocks always take the two-launch path
            // (also after the prefilter was switched off for not being selective)
            bool lazy_read_early = false;  // a lazy column holds cell references, not offsets: the prefilter must not load it
            if (lazy && s->prefilter)
                for (const tplx_instr &in : s->prefilter->instrs)
                    if (in.op == TPLX_OP_LDCOL && (size_t)in.imm < b->mapped.size() && b->mapped[in.imm] == 2) lazy_read_early = true;
            if (lazy && !s->prefilter)
                rc = fail(TPLX_E_UNSUPPORTED, "stage_run: block has lazy CSV columns but the stage has no prefilter; parse without col_lazy");
            else if (lazy_read_early)
                rc = fail(TPLX_E_BADARG, "stage_run: a column parsed with col_lazy is read by the stage's prefilter; parse it eagerly");
            else
                rc = (s->prefilter && (s->prefilter_enabled.load(relaxed) || lazy)) ? run_rows_prefiltered(s, sd, b, first_row_no, r)
                                                                        : run_rows(s, sd, b, first_row_no, r, nullptr, 0);
            break;
        }
        case TPLX_EP_AGGREGATE:
        default: {
            bool lazy = false;
            for (uint8_t m : b->mapped) lazy = lazy || m == 2;
            if (lazy) rc = fail(TPLX_E_UNSUPPORTED, "stage_run: lazy CSV columns need a row stage with a prefilter");
            else rc = s->hdr.endpoint == TPLX_EP_AGGREGATE ? run_agg(s, sd, b, r) : run_hash(s, sd, b, r);
            break;
        }
    }
    if (rc) {
        tplx_gpu_result_free(r);
        return rc;
    }
    CU(cudaEventRecord(r->ev1, d->stream));
    *out = r;
    return TPLX_OK;
}

extern "C" int32_t tplx_gpu_stage_run_host(tplx_stage *s, int32_t device, const tplx_column *cols, uint32_t n_cols,
                                           uint64_t n_rows, int64_t first_row_no, tplx_result **out) {
    Device *d = get_device(device);
    if (!d) return fail(TPLX_E_NODEVICE, "stage_run_host: device not initialised (no CPU fallback)");
    CU(cudaSetDevice(d->id));
    cudaEvent_t e0;
    CU(cudaEventCreate(&e0));
    CU(cudaEventRecord(e0, d->copy_stream));  // the upload runs on the copy stream
    tplx_block *b = nullptr;
    int32_t rc = TPLX_OK;
    uint64_t h2d = 0;
    uint32_t zc = 0;
    if (s && s->prefilter && s->prefilter_enabled.load(relaxed) && s->hdr.endpoint == TPLX_EP_MEMORY && cols && n_cols == s->in_types.size() && !s->n_companions) {
        // Late materialisation across PCIe: only the columns the prefilter reads are copied to HBM. The other
        // columns are needed for surviving rows only; when they lie in page-locked host memory the dense launch
        // reads exactly those rows through the mapped address (zero-copy), otherwise they are copied like before.
        std::vector<bool> early(n_cols, false);
        for (const tplx_instr &in : s->prefilter->instrs)
            if (in.op == TPLX_OP_LDCOL) early[in.imm] = true;
        std::vector<tplx_column> up;       // columns to copy
        std::vector<uint32_t> up_idx;
        std::vector<ColIn> mapped(n_cols);
        std::vector<bool> is_mapped(n_cols, false);
        for (uint32_t c = 0; c < n_cols; ++c) {
            bool zero_copy = false;
            if (!early[c] && n_rows) {
                cudaPointerAttributes at{}, ao{};
                bool ok = cudaPointerGetAttributes(&at, cols[c].data) == cudaSuccess && at.type == cudaMemoryTypeHost && at.devicePointer;
                if (ok && cols[c].type == TPLX_T_STR)
                    ok = cudaPointerGetAttributes(&ao, cols[c].offsets) == cudaSuccess && ao.type == cudaMemoryTypeHost && ao.devicePointer;
                cudaGetLastError();
                if (ok) {
                    mapped[c].type = cols[c].type;
                    mapped[c].data = at.devicePointer;
                    mapped[c].offsets = cols[c].type == TPLX_T_STR ? static_cast<const uint32_t *>(ao.devicePointer) : nullptr;
                    zero_copy = true;
                }
            }
            if (zero_copy) { is_mapped[c] = true; ++zc; }
            else { up.push_back(cols[c]); up_idx.push_back(c); }
        }
        tplx_block *ub = nullptr;
        rc = tplx_gpu_block_upload(device, up.data(), (uint32_t)up.size(), n_rows, &ub);
        if (rc) { cudaEventDestroy(e0); return rc; }
        b = new tplx_block();
        b->dev = d;
        b->n_rows = n_rows;
        b->cols.resize(n_cols);
        b->data_bytes.resize(n_cols);
        for (size_t k = 0; k < up_idx.size(); ++k) {
            b->cols[up_idx[k]] = ub->cols[k];
            b->data_bytes[up_idx[k]] = ub->data_bytes[k];
            h2d += ub->data_bytes[k] + (up[k].type == TPLX_T_STR ? (n_rows + 1) * 4 : 0);
        }
        b->mapped.assign(n_cols, 0);
        for (uint32_t c = 0; c < n_cols; ++c)
            if (is_mapped[c]) {
                b->mapped[c] = 1;
                b->cols[c] = mapped[c];
                b->data_bytes[c] = cols[c].type == TPLX_T_STR ? cols[c].data_bytes : n_rows * 8;
            }
        b->owned = ub->owned;
        b->ready = ub->ready;
        ub->owned.clear();
        delete ub;
    } else {
        rc = tplx_gpu_block_upload(device, cols, n_cols, n_rows, &b);
        if (rc) { cudaEventDestroy(e0); return rc; }
        for (uint32_t c = 0; c < n_cols; ++c)
            h2d += (cols[c].type == TPLX_T_STR ? cols[c].data_bytes + (n_rows + 1) * 4 : n_rows * 8);
    }
    rc = tplx_gpu_stage_run(s, b, first_row_no, out);
    if (rc) {
        tplx_gpu_block_free(b);
        cudaEventDestroy(e0);
        return rc;
    }
    cudaEventDestroy((*out)->ev0);
    (*out)->ev0 = e0;  // total time includes the H2D copies
    (*out)->owned_block = b;
    (*out)->h2d_bytes = h2d;
    (*out)->zero_copy_cols = zc;
    return TPLX_OK;
}

static int32_t fill_common(KParams &P, tplx_stage *s, StageDev *sd, const tplx_block *b, const Layout &L, uint32_t R) {
    memset(&P, 0, sizeof(P));
    P.n_rows = b->n_rows;
    P.n_instr = (uint32_t)s->instrs.size();
    P.n_slots = s->hdr.n_slots;
    P.n_in = (uint32_t)s->in_types.size();
    P.n_out = (uint32_t)s->out_cols.size();
    P.n_str_out = s->n_str_out;
    P.n_accs = (uint32_t)s->accs.size();
    P.R = R;
    P.n_work = b->n_rows;
    P.rowlist = nullptr;
    P.n_tiles = (uint32_t)((b->n_rows + (uint64_t)R * NT - 1) / ((uint64_t)R * NT));
    P.K = 2 + s->n_str_out;
    P.smem_cols_off = L.cols_off;
    P.smem_regs_off = L.regs_off;
    P.smem_stage_off = L.stage_off;
    P.smem_misc_off = L.misc_off;
    P.smem_stash_off = L.stash_off;
    P.inplace = L.inplace ? 1u : 0u;
    P.prog = sd->prog;
    P.cpool = sd->cpool;
    P.opids = sd->opids;
    for (size_t c = 0; c < b->cols.size(); ++c) P.in[c] = b->cols[c];
    for (size_t k = 0; k < s->accs.size(); ++k) {
        P.accs[k].kind = s->accs[k].kind;
        P.accs[k].slot = s->accs[k].slot;
        P.accs[k].init = s->accs[k].init;
    }
    return TPLX_OK;
}

template <typename T>
static int32_t dalloc(tplx_result *r, T **p, size_t count) {
    void *q = nullptr;
    CU(cudaMallocAsync(&q, std::max<size_t>(count * sizeof(T), 16), r->dev->stream));
    r->owned.push_back(q);
    *p = static_cast<T *>(q);
    return TPLX_OK;
}

// lens[0 .. n) = string lengths, in place to their exclusive scan; *total = lens[n], fetched with a synchronise. A total beyond 32-bit
// offsets fails with `what`.
static int32_t str_total(Device *d, uint64_t *lens, uint64_t n, uint64_t *total, const char *what) {
    int32_t rc = device_scan(d, lens, lens, n, true);
    if (rc) return rc;
    CU(cudaMemcpyAsync(total, lens + n, 8, cudaMemcpyDeviceToHost, d->stream));
    CU(cudaStreamSynchronize(d->stream));
    if (*total > 0xFFFFFFFFull) return fail(TPLX_E_OVERFLOW, what);
    return TPLX_OK;
}

// Events of a result made outside stage_run (join probe, merge, hash export), from which tplx_gpu_result_info derives kernel_ms and
// total_ms: result_begin after the input block `in` (may be null) is ready, result_end when all work is enqueued.
static int32_t result_begin(tplx_result *r, const tplx_block *in) {
    Device *d = r->dev;
    CU(cudaEventCreate(&r->ev0));
    CU(cudaEventCreate(&r->ev1));
    CU(cudaEventCreate(&r->evk0));
    CU(cudaEventCreate(&r->evk1));
    if (in && in->ready) CU(cudaStreamWaitEvent(d->stream, in->ready, 0));
    CU(cudaEventRecord(r->ev0, d->stream));
    CU(cudaEventRecord(r->evk0, d->stream));
    return TPLX_OK;
}
static int32_t result_end(tplx_result *r) {
    Device *d = r->dev;
    CU(cudaGetLastError());
    CU(cudaEventRecord(r->evk1, d->stream));
    CU(cudaEventRecord(r->ev1, d->stream));
    CU(cudaStreamSynchronize(d->stream));
    return TPLX_OK;
}

// Output column `oc` of r (type r->out_types[oc]) from n rows picked by `sel` out of sources a and b (gather.cuh). A validity bitmap
// is made when force_valid or a source has one. Launches: 5 for a string column, 1 for fixed width, +1 for a bitmap. `what` is the
// error message of a string column beyond 4 GiB.
static int32_t gather_column(tplx_result *r, size_t oc, SelSrc a, SelSrc b, uint32_t b_bit, const uint32_t *sel, uint64_t n, bool force_valid,
                             const char *what) {
    Device *d = r->dev;
    const uint32_t nb = (uint32_t)((n + SEL_NT - 1) / SEL_NT);
    int32_t rc;
    if (r->out_types[oc] == TPLX_T_STR) {
        uint64_t *lens = nullptr, tot = 0;
        CU(cudaMallocAsync((void **)&lens, (n + 1) * 8, d->stream));
        if (n) sel_str_len_kernel<<<nb, SEL_NT, 0, d->stream>>>(a, b, b_bit, sel, n, lens);
        rc = str_total(d, lens, n, &tot, what);
        if (!rc) rc = dalloc(r, &r->out[oc].offsets, n + 1);
        if (!rc) rc = dalloc(r, &r->out[oc].bytes, str_buf_bytes(tot));
        if (!rc)
            sel_str_copy_kernel<<<(uint32_t)(((n + 1) * SEL_STR_LANES + SEL_NT - 1) / SEL_NT), SEL_NT, 0, d->stream>>>(
                a, b, b_bit, sel, n, lens, r->out[oc].offsets, r->out[oc].bytes);
        cudaFreeAsync(lens, d->stream);
        if (rc) return rc;
        r->out[oc].cap_bytes = tot;
        r->str_bytes[oc] = tot;
        r->launches += 5;
    } else {
        if ((rc = dalloc(r, &r->out[oc].data, n))) return rc;
        if (n) sel_gather_fixed_kernel<<<nb, SEL_NT, 0, d->stream>>>(a, b, b_bit, sel, n, r->out[oc].data);
        r->launches += 1;
    }
    if (force_valid || a.valid || b.valid) {
        if ((rc = dalloc(r, &r->out_valid[oc], (n + 31) / 32 + 1))) return rc;
        if (n) sel_gather_valid_kernel<<<nb, SEL_NT, 0, d->stream>>>(a, b, b_bit, sel, n, r->out_valid[oc]);
        r->launches += 1;
    }
    CU(cudaGetLastError());
    return TPLX_OK;
}

// K1v (vecvm.cuh): fixed-width stages, vector-at-a-time. Outputs are fixed width, so capacities are exact (n rows) and the only
// retry is for exception records.
template <int J>
static int32_t launch_rows_vec(uint32_t grid, uint32_t smem, cudaStream_t st, const KParams &P) {
    CU(cudaFuncSetAttribute(stage_rows_vec_kernel<J>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    stage_rows_vec_kernel<J><<<grid, NT, smem, st>>>(P);
    return TPLX_OK;
}
static int32_t run_rows_vec(tplx_stage *s, StageDev *sd, const tplx_block *b, int64_t first_row_no, tplx_result *r) {
    Device *d = r->dev;
    const uint64_t n = b->n_rows;
    const uint32_t ns = s->vplan.n_slots;
    const size_t n_uops = s->vplan.ins.size();
    // J = 4 (2048-row tiles, 8 rows per thread per dispatch) when the register file leaves room for >= 3 CTAs per SM, else J = 2
    int Jsel = 0;
    uint32_t T = 0;
    Layout L;
    for (int J : {4, 2}) {
        T = 2u * J * NT;
        L = vec_layout(s, std::max<size_t>(n_uops, 1) * sizeof(VInstr), T, (size_t)ns * T * 8, true);
        if (L.total <= 72 * 1024 || (J == 2 && L.total <= (uint32_t)d->smem_optin)) { Jsel = J; break; }
    }
    // specialised kernels (jit.inl), whose register file holds the live-out slots only: K1r (nothing staged, the tile is evaluated
    // again from L2 once its offset is known) for programs of a few operations; else K1w (4 sub-batches of 2048 rows per ticket) when
    // the live-out slots fit the shared memory of 3 resident CTAs; else K1v with J = 4 (8 rows per thread) when that fits, else J = 2.
    // While one of them is still compiling the interpreting kernel runs, and no second compile starts.
    jit::Loaded *jf = nullptr;
    if (jit_wanted(s, n)) {
        const uint32_t nl = std::max<uint32_t>((uint32_t)s->jit_live.slots.size(), 1);
        bool pending = false;
        auto take = [&](int kind, int J, uint32_t Tk, const Layout &Lk) {
            jf = jit_get(s, sd, kind, jit_minb(s, kind));
            if (jf) { Jsel = J; T = Tk; L = Lk; }
            else pending = jit_pending(s, kind);
        };
        if (s->instrs.size() <= 16) take(jit::K_RE2, 4, 2 * 2048u, vec_layout(s, 16, 2 * 2048u, 0, false));
        if (!jf && !pending) {
            const Layout Lw = vec_layout(s, 16, 4 * 2048u, (size_t)nl * 4 * 2048 * 8, false);
            if (Lw.total <= 74u * 1024) take(jit::K_WIDE4, 4, 4 * 2048u, Lw);
        }
        for (int J : {4, 2}) {
            if (jf || pending) break;
            const uint32_t Tj = 2u * J * NT;
            const Layout Lj = vec_layout(s, 16, Tj, (size_t)nl * Tj * 8, true);
            if (Lj.total > (J == 4 ? 56u * 1024 : 100u * 1024)) continue;
            take(J == 4 ? jit::K_VEC4 : jit::K_VEC2, J, Tj, Lj);
            break;
        }
    }
    if (!Jsel) return TPLX_E_UNSUPPORTED;
    const uint32_t smem = L.total;
    const int ji = Jsel == 4 ? 1 : 0;
    DInstr *prog_vec = nullptr;
    {  // built by the first block that needs it; both lanes may get here at once, so it is read under the lock too
        std::lock_guard<std::mutex> lk(s->mu);
        if (!jf && !sd->prog_vec[ji]) {
            std::vector<VInstr> dec = vec_encode(s->vplan, T, L.regs_off);
            VInstr *p = nullptr;
            CU(cudaMalloc(&p, std::max<size_t>(dec.size() * sizeof(VInstr), 16)));
            CU(cudaMemcpy(p, dec.data(), dec.size() * sizeof(VInstr), cudaMemcpyHostToDevice));
            sd->prog_vec[ji] = reinterpret_cast<DInstr *>(p);
        }
        prog_vec = sd->prog_vec[ji];
    }
    KParams P;
    fill_common(P, s, sd, b, L, 2 * Jsel);
    P.prog = prog_vec;
    P.n_instr = jf ? 0u : (uint32_t)n_uops;
    P.n_slots = jf ? (uint32_t)s->jit_live.slots.size() : ns;

    P.n_tiles = (uint32_t)((n + T - 1) / T);
    P.first_row_no = first_row_no;
    int occ = 0;
    if (jf) occ = jit_occupancy(jf, smem);
    else if (Jsel == 4) {
        CU(cudaFuncSetAttribute(stage_rows_vec_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, stage_rows_vec_kernel<4>, NT, smem));
    } else {
        CU(cudaFuncSetAttribute(stage_rows_vec_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, stage_rows_vec_kernel<2>, NT, smem));
    }
    if (occ < 1) return TPLX_E_UNSUPPORTED;
    const uint32_t grid = std::max<uint32_t>(1, std::min<uint32_t>(P.n_tiles, (uint32_t)(occ * d->prop.multiProcessorCount)));
    r->hidden = s->hidden;
    r->out_types.clear();
    for (auto &oc : s->out_cols) r->out_types.push_back(oc.type);
    r->str_bytes.assign(s->out_cols.size(), 0);
    r->out.assign(s->out_cols.size(), OutCol{});
    CU(cudaEventRecord(r->evk0, d->stream));
    if (n == 0) {
        CU(cudaEventRecord(r->evk1, d->stream));
        return TPLX_OK;
    }
    uint64_t *tile_state = nullptr, *totals = nullptr;
    uint32_t *counters = nullptr;
    KParams *dP = nullptr;
    const size_t state_words = (size_t)P.n_tiles;  // one packed word per tile (vec_tile_finish)
    int32_t rc = dalloc(r, &tile_state, state_words);
    if (rc) return rc;
    rc = dalloc(r, &totals, MAX_SCAN);
    if (rc) return rc;
    rc = dalloc(r, &counters, 4);
    if (rc) return rc;
    rc = dalloc(r, &dP, 1);
    if (rc) return rc;
    P.tile_state = tile_state;
    P.totals = totals;
    P.counters = counters;
    for (size_t c = 0; c < s->out_cols.size(); ++c) {
        OutCol &oc = P.out[c];
        oc.slot = s->out_cols[c].slot;
        oc.type = s->out_cols[c].type;
        oc.strk = -1;
        oc.stage_off = (jf ? (uint32_t)s->jit_live.map[s->out_cols[c].slot] : (uint32_t)s->vplan.slot_map[s->out_cols[c].slot]) * T * 8;
        rc = dalloc(r, &oc.data, n);
        if (rc) return rc;
    }
    P.cap_rows = n;
    uint64_t cap_exc = std::max<uint64_t>(4096, (uint64_t)(s->est_exc_per_row.load(relaxed) * 1.5 * (double)n) + n / 64);
    for (int attempt = 0; attempt < 2; ++attempt) {
        P.cap_exc = cap_exc;
        rc = dalloc(r, &P.exc, cap_exc);
        if (rc) return rc;
        CU(cudaMemsetAsync(tile_state, 0, state_words * 8, d->stream));
        CU(cudaMemsetAsync(counters, 0, 16, d->stream));
        CU(cudaMemsetAsync(totals, 0, MAX_SCAN * 8, d->stream));
        rc = jf ? jit_launch(jf, grid, smem, d->stream, &P) : Jsel == 4 ? launch_rows_vec<4>(grid, smem, d->stream, P) : launch_rows_vec<2>(grid, smem, d->stream, P);
        if (rc) return rc;
        if (jf) r->jit_launches += 1;
        CU(cudaGetLastError());
        r->launches += 1;
        uint64_t h_tot[MAX_SCAN];
        uint32_t h_cnt[4];
        CU(cudaMemcpyAsync(h_tot, totals, MAX_SCAN * 8, cudaMemcpyDeviceToHost, d->stream));
        CU(cudaMemcpyAsync(h_cnt, counters, 16, cudaMemcpyDeviceToHost, d->stream));
        CU(cudaStreamSynchronize(d->stream));
        r->n_out = h_tot[0];
        r->n_exc = h_tot[1];
        s->est_exc_per_row.store((double)r->n_exc / (double)n, relaxed);
        if (h_cnt[1] == 0) break;
        if (attempt == 1) return fail(TPLX_E_OVERFLOW, "exception capacity retry failed");
        cap_exc = r->n_exc + 16;
    }
    CU(cudaEventRecord(r->evk1, d->stream));
    for (size_t c = 0; c < s->out_cols.size(); ++c) r->out[c] = P.out[c];
    r->exc = P.exc;
    return TPLX_OK;
}

// n_work_dev != nullptr: n_list is only the CAPACITY of the survivor list (an estimate); the real length is read on the device.
// Returns TPLX_INTERNAL_RETRY when the real length turned out larger (nothing usable was produced).
static int32_t run_rows(tplx_stage *s, StageDev *sd, const tplx_block *b, int64_t first_row_no, tplx_result *r,
                        const uint64_t *rowlist, uint64_t n_list, const std::vector<ColIn> *cols_override, const uint64_t *n_work_dev) {
    Device *d = r->dev;  // execution lane chosen by tplx_gpu_stage_run
    const uint64_t n = rowlist ? n_list : b->n_rows;  // rows to evaluate
    r->hidden = s->hidden;
    r->out_types.clear();
    for (auto &oc : s->out_cols) r->out_types.push_back(oc.type);
    r->str_bytes.assign(s->out_cols.size(), 0);
    r->out.assign(s->out_cols.size(), OutCol{});
    if (n == 0) {
        CU(cudaEventRecord(r->evk0, d->stream));
        CU(cudaEventRecord(r->evk1, d->stream));
        for (size_t c = 0; c < s->out_cols.size(); ++c)
            if (s->out_cols[c].type == TPLX_T_STR) {
                int32_t rc = dalloc(r, &r->out[c].offsets, 1);
                if (rc) return rc;
                CU(cudaMemsetAsync(r->out[c].offsets, 0, 4, d->stream));
            }
        return TPLX_OK;
    }
    if (s->vec_ok && !rowlist && !cols_override && !getenv("TPLX_NO_VEC") && b->n_rows < (1ull << 31)) {
        bool ok = true;
        for (size_t c = 0; c < b->cols.size(); ++c)
            ok = ok && !(b->cols[c].type & COL_COMPACT) && (c >= b->mapped.size() || !b->mapped[c]) && (((uintptr_t)b->cols[c].data & 15) == 0);
        if (ok) {
            int32_t vrc = run_rows_vec(s, sd, b, first_row_no, r);
            if (vrc != TPLX_E_UNSUPPORTED) return vrc;  // does not fit the vector kernel's shared memory: scalar kernel below
        }
    }
    // tile shape: the largest tile (fewest barrier / look-back episodes, best load balance inside the CTA) that does
    // not cost occupancy: the register-limited number of resident CTAs divides the SM's shared memory into budgets
    // specialised K1 (jit.inl): same kernel source around the generated row function, compact register file
    jit::Loaded *jf = nullptr;
    if (jit_wanted(s, b->n_rows)) {
        jf = jit_get(s, sd, jit::K_ROWS, jit_minb(s, jit::K_ROWS));
    }
    int occ_regs = 0;
    if (jf) occ_regs = jit_occupancy(jf, 0);
    else CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_regs, stage_rows_kernel, NT, 0));
    occ_regs = std::max(occ_regs, 1);
    uint32_t smem_budget = (uint32_t)(d->prop.sharedMemPerMultiprocessor / occ_regs) - 1024;
    uint32_t R = 16;
    Layout L = make_layout(s, R, true, false, jf != nullptr);
    while (R > 1 && L.total > smem_budget) {
        R /= 2;
        L = make_layout(s, R, true, true, jf != nullptr);  // one row per thread: no staging area, outputs are read from the register file
    }
    if (L.total > smem_budget && !(L.inplace && L.total <= (uint32_t)d->smem_optin)) {
        // even one row per thread does not fit the budget: give up occupancy instead
        smem_budget = (uint32_t)std::min<int>(d->smem_optin, 113 * 1024);
        R = 4;
        L = make_layout(s, R, true, false, jf != nullptr);
        while (R > 1 && L.total > smem_budget) {
            R /= 2;
            L = make_layout(s, R, true, true, jf != nullptr);
        }
    }
    if (L.total > (uint32_t)d->smem_optin) return fail(TPLX_E_UNSUPPORTED, "stage needs more shared memory than one SM has");
    int occ = 0;
    if (jf) occ = jit_occupancy(jf, L.total);
    else CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, stage_rows_kernel, NT, L.total));
    if (occ < 1) return fail(TPLX_E_UNSUPPORTED, "stage kernel cannot be resident");
    // String stages read their input bytes through L1 again and again (every string op walks the bytes): shared memory must not
    // take the whole 256 KB of the SM's L1 / shared memory. The carve-out is capped at 196 KB (85 % of 228), which leaves 60 KB of
    // L1 at 3 CTAs/SM, and occupancy is counted against it.
    const int carve = s->has_str ? 85 : -1;
    if (jf) jit::cudrv_api()->FuncSetAttribute(jf->fn, jit::CU_FUNC_ATTRIBUTE_PREFERRED_SHARED_MEMORY_CARVEOUT, carve);
    else CU(cudaFuncSetAttribute(stage_rows_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, carve));
    if (carve > 0 && carve < 100) {
        static const int steps_kb[] = {8, 16, 32, 64, 100, 132, 164, 196, 228};
        int cfg = 228;
        for (int kb : steps_kb)
            if (kb * 100 >= carve * 228) { cfg = kb; break; }
        occ = std::max(1, std::min(occ, (int)((size_t)cfg * 1024 / ((size_t)L.total + 1024))));
    }
    if (getenv("TPLX_TRACE"))
        fprintf(stderr, "[tplx] rows kernel%s: R %u, shared memory %u B (%s), %d CTAs/SM\n", jf ? " (specialised)" : "", R, L.total, L.inplace ? "in place" : "staged", occ);
    KParams P;
    fill_common(P, s, sd, b, L, R);
    if (jf) {
        P.n_instr = 0;
        P.n_slots = (uint32_t)s->jit_live.slots.size();
    }
    if (cols_override)
        for (size_t c = 0; c < cols_override->size(); ++c) P.in[c] = (*cols_override)[c];
    P.rowlist = rowlist;
    P.n_work = n;
    P.n_work_dev = n_work_dev;
    P.n_tiles = (uint32_t)((n + (uint64_t)R * NT - 1) / ((uint64_t)R * NT));
    const uint32_t grid = std::min<uint32_t>(P.n_tiles, (uint32_t)(occ * d->prop.multiProcessorCount));
    P.first_row_no = first_row_no;
    P.scratch_per_thread = s->materialises ? std::max<uint32_t>(s->hdr.scratch_bytes, 64) * R : 0;
    int32_t rc = ensure_scratch(d, (size_t)grid * NT * P.scratch_per_thread);
    if (rc) return rc;
    P.scratch = d->scratch;

    // capacities: rows worst case; string bytes + exceptions adaptive with exact retry
    uint64_t in_str_bytes = 0;
    for (size_t c = 0; c < b->cols.size(); ++c)
        if (s->in_types[c] == TPLX_T_STR) in_str_bytes += b->data_bytes[c];
    std::vector<uint64_t> cap_bytes(s->out_cols.size(), 0);
    for (size_t c = 0; c < s->out_cols.size(); ++c) {
        if (s->out_cols[c].type != TPLX_T_STR) continue;
        const double est = s->est_bytes_per_row[c].load(relaxed);
        uint64_t cap = est >= 0 ? (uint64_t)(est * 1.25 * (double)n) + (1u << 16) : in_str_bytes / 8 + n + (1u << 20);
        cap_bytes[c] = std::min<uint64_t>(cap, 0xFFFFFFFFull);
    }
    uint64_t cap_exc = std::max<uint64_t>(4096, (uint64_t)(s->est_exc_per_row.load(relaxed) * 1.5 * (double)n) + n / 64);
    uint64_t cap_rows = n;

    uint64_t *tile_state = nullptr, *totals = nullptr;
    uint32_t *counters = nullptr;
    KParams *dP = nullptr;
    const size_t state_words = (size_t)P.n_tiles * (1 + 2 * P.K);
    rc = dalloc(r, &tile_state, state_words);
    if (rc) return rc;
    rc = dalloc(r, &totals, MAX_SCAN);
    if (rc) return rc;
    rc = dalloc(r, &counters, 4);
    if (rc) return rc;
    rc = dalloc(r, &dP, 1);
    if (rc) return rc;
    P.tile_state = tile_state;
    P.totals = totals;
    P.counters = counters;

    for (int attempt = 0; attempt < 3; ++attempt) {
        int si = 0;
        for (size_t c = 0; c < s->out_cols.size(); ++c) {
            OutCol &oc = P.out[c];
            oc.slot = jf ? (uint32_t)s->jit_live.map[s->out_cols[c].slot] : s->out_cols[c].slot;
            oc.type = s->out_cols[c].type;
            oc.stage_off = L.col_stage_off[c];
            if (oc.type == TPLX_T_STR) {
                oc.strk = si++;
                oc.cap_bytes = cap_bytes[c];
                rc = dalloc(r, &oc.offsets, cap_rows + 1);
                if (rc) return rc;
                rc = dalloc(r, &oc.bytes, str_buf_bytes(cap_bytes[c]));
                if (rc) return rc;
                oc.data = nullptr;
            } else {
                oc.strk = -1;
                rc = dalloc(r, &oc.data, cap_rows);
                if (rc) return rc;
            }
        }
        P.cap_rows = cap_rows;
        P.cap_exc = cap_exc;
        rc = dalloc(r, &P.exc, cap_exc);
        if (rc) return rc;
        CU(cudaMemsetAsync(tile_state, 0, state_words * 8, d->stream));
        CU(cudaMemsetAsync(counters, 0, 16, d->stream));
        CU(cudaMemsetAsync(totals, 0, MAX_SCAN * 8, d->stream));
        CU(cudaEventRecord(r->evk0, d->stream));
        if (jf) {
            rc = jit_launch(jf, grid, L.total, d->stream, &P);
            if (rc) return rc;
            r->jit_launches += 1;
        } else stage_rows_kernel<<<grid, NT, L.total, d->stream>>>(P);
        CU(cudaGetLastError());
        CU(cudaEventRecord(r->evk1, d->stream));
        r->launches += 1;
        uint64_t h_tot[MAX_SCAN];
        uint32_t h_cnt[4];
        CU(cudaMemcpyAsync(h_tot, totals, MAX_SCAN * 8, cudaMemcpyDeviceToHost, d->stream));
        CU(cudaMemcpyAsync(h_cnt, counters, 16, cudaMemcpyDeviceToHost, d->stream));
        CU(cudaStreamSynchronize(d->stream));
        r->n_out = h_tot[0];
        r->n_exc = h_tot[1];
        // rows really evaluated (the device-side count when the host only had an estimate): the base of the per-row estimates
        const uint64_t n_act = n_work_dev ? std::max<uint64_t>(1, std::min<uint64_t>(d->pinned[0], n)) : n;
        si = 0;
        for (size_t c = 0; c < s->out_cols.size(); ++c)
            if (s->out_cols[c].type == TPLX_T_STR) {
                r->str_bytes[c] = h_tot[2 + si++];
                s->est_bytes_per_row[c].store((double)r->str_bytes[c] / (double)n_act, relaxed);
            }
        s->est_exc_per_row.store((double)r->n_exc / (double)n_act, relaxed);
        if (h_cnt[1] & 8u) return TPLX_INTERNAL_RETRY;  // more survivors than the estimate everything was sized for
        if (h_cnt[1] == 0) break;
        if (attempt == 2) return fail(TPLX_E_OVERFLOW, "output capacity retry failed");
        for (size_t c = 0; c < s->out_cols.size(); ++c)
            if (s->out_cols[c].type == TPLX_T_STR) {
                if (r->str_bytes[c] > 0xFFFFFFFFull)
                    return fail(TPLX_E_OVERFLOW, "string output column exceeds 4 GiB in one block; use smaller blocks");
                cap_bytes[c] = r->str_bytes[c] + 16;
            }
        cap_exc = r->n_exc + 16;
    }
    for (size_t c = 0; c < s->out_cols.size(); ++c) r->out[c] = P.out[c];
    r->exc = P.exc;
    return TPLX_OK;
}

// K1m (mask.cuh): the prefilter stage as a pure map -> bitmaps -> ascending survivor list + exception records.
// Fills ra like run_rows would for a row-index stage: ra->out[0].data = survivor list, ra->n_out, ra->exc, ra->n_exc.
// no_wait: nothing here blocks the host — the survivor list gets the worst-case capacity (n rows), the exception records an
// estimated one (*cap_exc_out), the counts stay on the device (*totals_dev: [0] survivors, [1] exception rows) and are also copied
// into the lane's page-locked buffer in stream order; the caller reads them after its own synchronisation.
static int32_t run_mask(tplx_stage *ps, StageDev *psd, const tplx_block *b, tplx_result *ra, bool no_wait, uint64_t **totals_dev, uint64_t *cap_exc_out) {
    Device *d = ra->dev;
    const uint64_t n = b->n_rows;
    ra->out.assign(1, OutCol{});
    ra->out_types.assign(1, TPLX_T_I64);
    ra->str_bytes.assign(1, 0);
    CU(cudaEventRecord(ra->evk0, d->stream));
    if (n == 0) {
        CU(cudaEventRecord(ra->evk1, d->stream));
        return TPLX_OK;
    }
    if (n > 0xFFFFFFFFull * 16) return fail(TPLX_E_UNSUPPORTED, "block too large for the mask stage");
    MaskParams P;
    memset(&P, 0, sizeof(P));
    P.n_rows = n;
    P.n_instr = (uint32_t)ps->instrs.size();
    // the stage's only output is the row index (LDROW): the bitmaps carry it, so the trailing load is not evaluated
    if (P.n_instr && ps->instrs.back().op == TPLX_OP_LDROW && ps->instrs.back().guard == TPLX_NOSLOT) P.n_instr -= 1;
    P.n_in = (uint32_t)ps->in_types.size();
    P.n_slots = std::max<uint32_t>(ps->hdr.n_slots, 1);
    // K1f: the planner stated the stage in closed form (string-scan hint) -> evaluate the terms directly, nothing is interpreted
    const bool scan = !ps->scan.empty() && !(getenv("TPLX_NO_SCAN") && atoi(getenv("TPLX_NO_SCAN")));
    // specialised K1m (jit.inl): for prefilters without a closed form
    jit::Loaded *jf = nullptr;
    if (!scan && jit_wanted(ps, n)) {
        jf = jit_get(ps, psd, jit::K_MASK, jit_minb(ps, jit::K_MASK));
        if (jf) {
            P.n_slots = 0;  // no register file: nothing is live out of a prefilter program
            P.n_instr = 0;
        }
    }
    if (scan) {
        P.n_terms = (uint32_t)ps->scan.size();
        memcpy(P.terms, ps->scan.data(), ps->scan.size() * sizeof(tplx_scan_term));
        P.n_slots = 0;  // no register file
        P.n_instr = 0;
    }
    P.n_tiles = (uint32_t)((n + 31) / 32);
    P.prog = psd->prog;
    P.cpool = psd->cpool;
    for (size_t c = 0; c < b->cols.size(); ++c) P.in[c] = b->cols[c];
    size_t off = align_up(std::max<size_t>(P.n_instr, 1) * sizeof(DInstr), 16);
    P.smem_regs_off = (uint32_t)off;
    off = align_up(off + (size_t)P.n_slots * NT * 8, 16);
    P.smem_cols_off = (uint32_t)off;
    const uint32_t smem_total = (uint32_t)align_up(off + std::max<uint32_t>(P.n_in, 1) * sizeof(ColIn), 16);
    if (smem_total > (uint32_t)d->smem_optin) return fail(TPLX_E_UNSUPPORTED, "mask stage needs more shared memory than one SM has");
    int occ = 0;
    if (jf) occ = jit_occupancy(jf, smem_total);
    else if (scan) CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, stage_mask_kernel<true>, NT, smem_total));
    else CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, stage_mask_kernel<false>, NT, smem_total));
    if (occ < 1) return fail(TPLX_E_UNSUPPORTED, "mask kernel cannot be resident");
    const uint32_t grid = std::max<uint32_t>(1, std::min<uint32_t>((P.n_tiles + MASK_WARPS - 1) / MASK_WARPS, (uint32_t)(occ * d->prop.multiProcessorCount)));
    P.scratch_per_thread = ps->materialises ? std::max<uint32_t>(ps->hdr.scratch_bytes, 64) : 0;
    int32_t rc = ensure_scratch(d, (size_t)grid * NT * P.scratch_per_thread);
    if (rc) return rc;
    P.scratch = d->scratch;
    const uint32_t n_words = P.n_tiles;
    const uint32_t nb = (n_words + CMP_NT - 1) / CMP_NT;
    uint64_t *part = nullptr, *totals = nullptr;
    rc = dalloc(ra, &P.keep_words, n_words);
    if (rc) return rc;
    rc = dalloc(ra, &P.exc_words, n_words);
    if (rc) return rc;
    rc = dalloc(ra, &P.exc_codes, n);
    if (rc) return rc;
    rc = dalloc(ra, &part, (size_t)nb * 2);
    if (rc) return rc;
    rc = dalloc(ra, &totals, 2);
    if (rc) return rc;
    if (jf) {
        rc = jit_launch(jf, grid, smem_total, d->stream, &P);
        if (rc) return rc;
        ra->jit_launches += 1;
    } else if (scan) stage_mask_kernel<true><<<grid, NT, smem_total, d->stream>>>(P);
    else stage_mask_kernel<false><<<grid, NT, smem_total, d->stream>>>(P);
    CU(cudaGetLastError());
    mask_count_kernel<<<nb, CMP_NT, 0, d->stream>>>(P.keep_words, P.exc_words, n_words, part);
    mask_scan_kernel<<<1, CMP_NT, 0, d->stream>>>(part, nb, totals);
    CU(cudaGetLastError());
    if (totals_dev) *totals_dev = totals;
    if (no_wait) {
        const uint64_t cap_exc = std::max<uint64_t>(4096, (uint64_t)(ps->est_exc_per_row.load(relaxed) * 1.5 * (double)n) + n / 64);
        if (cap_exc_out) *cap_exc_out = cap_exc;
        rc = dalloc(ra, &ra->out[0].data, n);  // worst case: every row survives
        if (rc) return rc;
        rc = dalloc(ra, &ra->exc, cap_exc);
        if (rc) return rc;
        mask_expand_kernel<<<nb, CMP_NT, 0, d->stream>>>(P.keep_words, P.exc_words, n_words, part, ra->out[0].data, P.exc_codes, psd->opids, ra->exc, cap_exc);
        CU(cudaGetLastError());
        CU(cudaMemcpyAsync(d->pinned, totals, 16, cudaMemcpyDeviceToHost, d->stream));
        ra->n_out = ra->n_exc = 0;  // filled in by the caller once the stream has been synchronised
    } else {
        uint64_t h_tot[2] = {0, 0};
        CU(cudaMemcpyAsync(h_tot, totals, 16, cudaMemcpyDeviceToHost, d->stream));
        CU(cudaStreamSynchronize(d->stream));
        ra->n_out = h_tot[0];
        ra->n_exc = h_tot[1];
        if (cap_exc_out) *cap_exc_out = ra->n_exc;
        rc = dalloc(ra, &ra->out[0].data, ra->n_out);
        if (rc) return rc;
        rc = dalloc(ra, &ra->exc, ra->n_exc);
        if (rc) return rc;
        mask_expand_kernel<<<nb, CMP_NT, 0, d->stream>>>(P.keep_words, P.exc_words, n_words, part, ra->out[0].data, P.exc_codes, psd->opids, ra->exc, ra->n_exc);
        CU(cudaGetLastError());
    }
    // kept for a later re-expansion (exception capacity exceeded in no_wait mode)
    ra->mask_keep = P.keep_words;
    ra->mask_exc = P.exc_words;
    ra->mask_codes = P.exc_codes;
    ra->mask_part = part;
    ra->mask_words = n_words;
    CU(cudaEventRecord(ra->evk1, d->stream));
    ra->launches += 4;
    return TPLX_OK;
}

// Selective pipelines: (1) prefilter stage over every row -> ascending list of surviving row indices,
// (2) this stage densely over that list. Exception rows of both launches are merged and numbered like one
// TransformTask would have numbered them (rows written + exceptions so far, TransformTask.cc:764,885).
static int32_t run_rows_prefiltered(tplx_stage *s, StageDev *sd, const tplx_block *b, int64_t first_row_no, tplx_result *r) {
    Device *d = r->dev;
    tplx_stage *ps = s->prefilter;
    StageDev *psd = nullptr;
    int32_t rc = stage_dev(ps, d, &psd);
    if (rc) return rc;
    tplx_result ra;
    ra.dev = d;
    ra.stage = ps;
    CU(cudaEventCreate(&ra.evk0));
    CU(cudaEventCreate(&ra.evk1));
    auto drop_ra = [&]() {
        for (void *p : ra.owned) cudaFreeAsync(p, d->stream);
        ra.owned.clear();
        if (ra.evk0) cudaEventDestroy(ra.evk0);
        if (ra.evk1) cudaEventDestroy(ra.evk1);
        ra.evk0 = ra.evk1 = nullptr;
    };
    struct OnExit {  // CU(...) early returns release the prefilter's temporaries too (drop_ra is idempotent)
        decltype(drop_ra) &f;
        ~OnExit() { f(); }
    } ra_guard{drop_ra};
    bool any_mapped = false;
    for (uint8_t m : b->mapped) any_mapped = any_mapped || m;
    // Steady state without a host round trip between the two launches: once a block has shown the selectivity, the dense launch of
    // the next block is sized from it (x1.3 + slack) and reads the real survivor count on the device; the host synchronises once,
    // at the end. (Blocks with late columns in host memory size their gather from the exact count and keep the round trip.)
    const double est_surv = ps->est_surv_ratio.load(relaxed);  // read once: the check and the sizing below see the same value
    const bool no_wait = !any_mapped && est_surv >= 0.0 && b->n_rows > 0 && !(getenv("TPLX_SYNC_PREFILTER") && atoi(getenv("TPLX_SYNC_PREFILTER")));
    uint64_t *totals_dev = nullptr, cap_exc_a = 0;
    rc = run_mask(ps, psd, b, &ra, no_wait, &totals_dev, &cap_exc_a);
    if (rc) { drop_ra(); return rc; }
    // the prefilter's kernel interval is timed lazily (result_info): no host synchronisation for it here
    r->extra_ev.emplace_back(ra.evk0, ra.evk1);
    ra.evk0 = ra.evk1 = nullptr;
    float msa = 0;
    if (no_wait) {
        const uint64_t cap = std::min<uint64_t>(b->n_rows, (uint64_t)(est_surv * 1.3 * (double)b->n_rows) + 65536);
        rc = run_rows(s, sd, b, first_row_no, r, ra.out[0].data, cap, nullptr, totals_dev);  // synchronises the stream at its end
        if (rc != TPLX_OK && rc != TPLX_INTERNAL_RETRY) { drop_ra(); return rc; }
        ra.n_out = d->pinned[0];
        ra.n_exc = d->pinned[1];
        ps->est_surv_ratio.store((double)ra.n_out / (double)b->n_rows, relaxed);
        ps->est_exc_per_row.store((double)ra.n_exc / (double)b->n_rows, relaxed);
        if (ra.n_exc > cap_exc_a) {  // more prefilter exceptions than estimated: expand them again with the exact capacity
            int32_t rc2 = dalloc(&ra, &ra.exc, ra.n_exc);
            if (rc2) { drop_ra(); return rc2; }
            const uint32_t nb = (ra.mask_words + CMP_NT - 1) / CMP_NT;
            uint64_t *dummy = nullptr;
            rc2 = dalloc(&ra, &dummy, ra.n_out + 1);
            if (rc2) { drop_ra(); return rc2; }
            mask_expand_kernel<<<nb, CMP_NT, 0, d->stream>>>(ra.mask_keep, ra.mask_exc, ra.mask_words, ra.mask_part, dummy, ra.mask_codes, psd->opids, ra.exc, ra.n_exc);
            CU(cudaGetLastError());
        }
        if (rc == TPLX_INTERNAL_RETRY) {  // more survivors than the estimate: the dense launch again, sized exactly
            for (void *p : r->owned) cudaFreeAsync(p, d->stream);
            r->owned.clear();
            r->launches = 0;
            rc = run_rows(s, sd, b, first_row_no, r, ra.out[0].data, ra.n_out, nullptr);
            if (rc) { drop_ra(); return rc; }
        }
        r->launches += ra.launches;
        r->jit_launches += ra.jit_launches;
    }
    const uint64_t n_surv = ra.n_out;
    if (!no_wait) {
        if (b->n_rows) {
            ps->est_surv_ratio.store((double)n_surv / (double)b->n_rows, relaxed);
            ps->est_exc_per_row.store((double)ra.n_exc / (double)b->n_rows, relaxed);
        }
    }
    if (b->n_rows >= (1u << 16) && n_surv * 2 > b->n_rows) s->prefilter_enabled.store(false, relaxed);  // not selective: stop using it
    // late columns that still live in host memory: bring over the surviving rows only (gather.cuh)
    std::vector<ColIn> dense_cols;
    float msg = 0;
    if (any_mapped && n_surv) {
        struct EvPair {  // released on every exit path
            cudaEvent_t a = nullptr, b = nullptr;
            ~EvPair() { if (a) cudaEventDestroy(a); if (b) cudaEventDestroy(b); }
        } gev;
        CU(cudaEventCreate(&gev.a));
        CU(cudaEventCreate(&gev.b));
        cudaEvent_t g0 = gev.a, g1 = gev.b;
        CU(cudaEventRecord(g0, d->stream));
        GatherCols G;
        memset(&G, 0, sizeof(G));
        std::vector<uint32_t> gcol;
        dense_cols.assign(b->cols.begin(), b->cols.end());
        for (uint32_t c = 0; c < b->cols.size(); ++c) {
            if (!b->mapped[c]) continue;
            const uint32_t k = G.n_cols++;
            gcol.push_back(c);
            G.type[k] = (uint8_t)b->cols[c].type;
            G.src_data[k] = b->cols[c].data;
            G.src_off[k] = b->cols[c].offsets;
            if (b->mapped[c] == 2) {
                G.src_ref[k] = reinterpret_cast<const uint64_t *>(b->cols[c].offsets);
                G.src_off[k] = nullptr;
                G.quote = b->csv_quote;
            }
            if (G.type[k] == TPLX_T_STR) {
                rc = dalloc(r, &G.lens[k], n_surv + 1);
                if (rc) { drop_ra(); return rc; }
                CU(cudaMemsetAsync(G.lens[k] + n_surv, 0, 8, d->stream));
                rc = dalloc(r, &G.srcpos[k], n_surv);
                if (rc) { drop_ra(); return rc; }
                rc = dalloc(r, &G.dst_off[k], n_surv + 1);
                if (rc) { drop_ra(); return rc; }
            } else {
                rc = dalloc(r, &G.dst_data[k], n_surv);
                if (rc) { drop_ra(); return rc; }
            }
        }
        GatherCols *dG = nullptr;
        rc = dalloc(r, &dG, 1);
        if (rc) { drop_ra(); return rc; }
        CU(cudaMemcpyAsync(dG, &G, sizeof(G), cudaMemcpyHostToDevice, d->stream));
        gather_pass1<<<(uint32_t)((n_surv + 255) / 256), 256, 0, d->stream>>>(ra.out[0].data, n_surv, dG);
        std::vector<uint64_t> totals(G.n_cols, 0);
        for (uint32_t k = 0; k < G.n_cols; ++k) {
            if (G.type[k] != TPLX_T_STR) continue;
            rc = device_scan(d, G.lens[k], G.lens[k], n_surv, true);
            if (rc) { drop_ra(); return rc; }
            CU(cudaMemcpyAsync(&totals[k], G.lens[k] + n_surv, 8, cudaMemcpyDeviceToHost, d->stream));
        }
        CU(cudaStreamSynchronize(d->stream));
        for (uint32_t k = 0; k < G.n_cols; ++k) {
            if (G.type[k] != TPLX_T_STR) continue;
            if (totals[k] > 0xFFFFFFFFull) { drop_ra(); return fail(TPLX_E_OVERFLOW, "gathered string column exceeds 4 GiB"); }
            rc = dalloc(r, &G.dst_bytes[k], str_buf_bytes(totals[k]));
            if (rc) { drop_ra(); return rc; }
        }
        CU(cudaMemcpyAsync(dG, &G, sizeof(G), cudaMemcpyHostToDevice, d->stream));
        gather_pass2<<<(uint32_t)(((n_surv + 1) * 32 + 255) / 256), 256, 0, d->stream>>>(n_surv, dG, ra.out[0].data);
        CU(cudaGetLastError());
        CU(cudaEventRecord(g1, d->stream));
        for (uint32_t k = 0; k < G.n_cols; ++k) {
            ColIn ci{};
            ci.type = (uint64_t)G.type[k] | COL_COMPACT;
            if (G.type[k] == TPLX_T_STR) { ci.data = G.dst_bytes[k]; ci.offsets = G.dst_off[k]; }
            else ci.data = G.dst_data[k];
            dense_cols[gcol[k]] = ci;
        }
        CU(cudaEventSynchronize(g1));
        CU(cudaEventElapsedTime(&msg, g0, g1));
        r->launches += 2 + 3 * G.n_cols;
    }
    if (!no_wait) {
        rc = run_rows(s, sd, b, first_row_no, r, ra.out[0].data, n_surv, dense_cols.empty() ? nullptr : &dense_cols);
        if (rc) { drop_ra(); return rc; }
        r->launches += ra.launches;
        r->jit_launches += ra.jit_launches;
    }
    r->kernel_ms_extra = msa + msg;
    const uint64_t na = ra.n_exc, nb = r->n_exc;
    if (na) {
        // stream-ordered copies: the lane's stream is non-blocking, so a plain cudaMemcpy would not wait for the kernels that wrote
        // these records (with no surviving row the dense launch — and its synchronisation — never happens)
        std::vector<tplx_exception_rec> ea(na), eb(nb), merged;
        CU(cudaMemcpyAsync(ea.data(), ra.exc, na * sizeof(tplx_exception_rec), cudaMemcpyDeviceToHost, d->stream));
        if (nb) CU(cudaMemcpyAsync(eb.data(), r->exc, nb * sizeof(tplx_exception_rec), cudaMemcpyDeviceToHost, d->stream));
        // input row index of every output row (hidden last column), ascending
        std::vector<int64_t> out_rows(r->n_out);
        if (r->n_out) CU(cudaMemcpyAsync(out_rows.data(), r->out.back().data, r->n_out * 8, cudaMemcpyDeviceToHost, d->stream));
        CU(cudaStreamSynchronize(d->stream));
        // B numbered its exceptions within its own stream: rows written before + index among B's exceptions
        for (uint64_t i = 0; i < nb; ++i) eb[i].row_no = eb[i].row_no - first_row_no - (int64_t)i;  // = rows written before
        for (uint64_t i = 0; i < na; ++i)
            ea[i].row_no = (int64_t)(std::lower_bound(out_rows.begin(), out_rows.end(), ea[i].row) - out_rows.begin());
        merged.resize(na + nb);
        std::merge(ea.begin(), ea.end(), eb.begin(), eb.end(), merged.begin(),
                   [](const tplx_exception_rec &x, const tplx_exception_rec &y) { return x.row < y.row; });
        for (uint64_t i = 0; i < merged.size(); ++i) merged[i].row_no += first_row_no + (int64_t)i;
        tplx_exception_rec *dm = nullptr;
        rc = dalloc(r, &dm, merged.size());
        if (rc) { drop_ra(); return rc; }
        CU(cudaMemcpyAsync(dm, merged.data(), merged.size() * sizeof(tplx_exception_rec), cudaMemcpyHostToDevice, d->stream));
        CU(cudaStreamSynchronize(d->stream));  // `merged` is a local
        r->exc = dm;
        r->n_exc = merged.size();
    }
    drop_ra();
    return TPLX_OK;
}

// K3f dispatch: smallest instantiation that holds the predicates / terms; padding entries are neutral
template <int NP, int NTM>
static int32_t launch_fused_tma_one(uint32_t sms, uint32_t n_tiles, uint32_t smem, cudaStream_t st, const KParams *dP, const FusedTmaParams *dF) {
    CU(cudaFuncSetAttribute(fused_scan_agg_tma_kernel<NP, NTM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 0;
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fused_scan_agg_tma_kernel<NP, NTM>, NT, smem));
    if (occ < 1) return fail(TPLX_E_UNSUPPORTED, "fused TMA kernel cannot be resident");
    const uint32_t grid = std::max<uint32_t>(1, std::min<uint32_t>(n_tiles, sms * (uint32_t)std::min(occ, 2)));
    fused_scan_agg_tma_kernel<NP, NTM><<<grid, NT, smem, st>>>(dP, dF);
    return TPLX_OK;
}
template <int NP>
static int32_t launch_fused_tma_np(uint32_t ntm, uint32_t sms, uint32_t n_tiles, uint32_t smem, cudaStream_t st, const KParams *dP, const FusedTmaParams *dF) {
    switch (ntm) {
        case 1: return launch_fused_tma_one<NP, 1>(sms, n_tiles, smem, st, dP, dF);
        case 2: return launch_fused_tma_one<NP, 2>(sms, n_tiles, smem, st, dP, dF);
        default: return launch_fused_tma_one<NP, 4>(sms, n_tiles, smem, st, dP, dF);
    }
}
template <int NP>
static int32_t launch_fused_np(uint32_t ntm, uint32_t grid, cudaStream_t st, const KParams *dP, const FusedParams *dF) {
    switch (ntm) {
        case 1: fused_scan_agg_kernel<NP, 1><<<grid, NT, 0, st>>>(dP, dF); break;
        case 2: fused_scan_agg_kernel<NP, 2><<<grid, NT, 0, st>>>(dP, dF); break;
        case 4: fused_scan_agg_kernel<NP, 4><<<grid, NT, 0, st>>>(dP, dF); break;
        default: fused_scan_agg_kernel<NP, 8><<<grid, NT, 0, st>>>(dP, dF); break;
    }
    return TPLX_OK;
}
static int32_t launch_fused(tplx_stage *s, Device *d, const KParams *dP, const KParams &P, tplx_result *r) {
    FusedParams F = s->fused;
    uint32_t np = F.n_preds <= 1 ? 1 : F.n_preds <= 2 ? 2 : F.n_preds <= 3 ? 3 : F.n_preds <= 4 ? 4 : 8;
    uint32_t ntm = F.n_terms <= 1 ? 1 : F.n_terms <= 2 ? 2 : F.n_terms <= 4 ? 4 : 8;
    if (F.n_terms > 8) return fail(TPLX_E_UNSUPPORTED, "fused scan: too many accumulators");
    const uint32_t some_col = F.n_preds ? F.preds[0].col : (F.terms[0].op != TPLX_FT_CONST ? F.terms[0].col_a : 0);
    // normalise predicates to inclusive ranges over ordered keys (see fused.cuh pred_pass)
    for (uint32_t i = 0; i < F.n_preds; ++i) {
        tplx_fused_pred &p = F.preds[i];
        const uint32_t fl = p.flags;
        int64_t lo = INT64_MIN, hi = INT64_MAX;
        if (fl & TPLX_FP_F64) {
            const int64_t kinf = f64_key(0x7FF0000000000000ull), kninf = f64_key(0xFFF0000000000000ull);
            lo = kninf;
            hi = kinf;  // NaN keys lie outside [-inf, +inf]: ordered compares with NaN are false
            if (fl & TPLX_FP_HAS_LO) {
                double v; memcpy(&v, &p.lo, 8);
                if (v != v) { lo = 1; hi = 0; }  // comparison against NaN is never true
                else { lo = f64_key((uint64_t)p.lo); if (!(fl & TPLX_FP_LO_INCL)) lo = lo == INT64_MAX ? lo : lo + 1; if (lo < kninf) lo = kninf; }
            }
            if ((fl & TPLX_FP_HAS_HI) && lo <= hi) {
                double v; memcpy(&v, &p.hi, 8);
                if (v != v) { lo = 1; hi = 0; }
                else { hi = f64_key((uint64_t)p.hi); if (!(fl & TPLX_FP_HI_INCL)) hi = hi == INT64_MIN ? hi : hi - 1; if (hi > kinf) hi = kinf; }
            }
            p.flags = (fl & TPLX_FP_CAST) ? 2 : 1;
        } else {
            if (fl & TPLX_FP_HAS_LO) { lo = p.lo; if (!(fl & TPLX_FP_LO_INCL)) { if (lo == INT64_MAX) { lo = 1; hi = 0; } else lo += 1; } }
            if ((fl & TPLX_FP_HAS_HI) && lo <= hi) { hi = p.hi; if (!(fl & TPLX_FP_HI_INCL)) { if (hi == INT64_MIN) { lo = 1; hi = 0; } else hi -= 1; } }
            p.flags = 0;
        }
        p.lo = lo;
        p.hi = hi;
    }
    for (uint32_t i = F.n_preds; i < np; ++i) { F.preds[i].col = some_col; F.preds[i].flags = 0; F.preds[i].lo = INT64_MIN; F.preds[i].hi = INT64_MAX; }
    for (uint32_t i = F.n_terms; i < ntm; ++i) { F.terms[i] = tplx_fused_term{}; F.terms[i].kind = TPLX_ACC_SUM_I64; F.terms[i].op = TPLX_FT_CONST; }
    if (P.n_in == 0) return fail(TPLX_E_UNSUPPORTED, "fused scan without input columns");
    // TMA-staged variant when the distinct columns fit the ring and every column base is 16-byte aligned
    if (!getenv("TPLX_NO_TMA") && ntm <= 4 && np <= 4) {
        FusedTmaParams FT;
        memset(&FT, 0, sizeof(FT));
        FT.f = F;
        bool ok = true;
        auto ucol_of = [&](uint32_t col) -> uint32_t {
            for (uint32_t i = 0; i < FT.n_ucols; ++i)
                if (FT.ucol[i] == col) return i;
            if (FT.n_ucols == TMA_MAX_UCOLS) { ok = false; return 0; }
            FT.ucol[FT.n_ucols] = col;
            return FT.n_ucols++;
        };
        for (uint32_t i = 0; i < np; ++i) FT.f.preds[i].col = ucol_of(F.preds[i].col);
        for (uint32_t i = 0; i < ntm; ++i) {
            if (F.terms[i].op != TPLX_FT_CONST) FT.f.terms[i].col_a = ucol_of(F.terms[i].col_a);
            if (F.terms[i].op == TPLX_FT_MUL) FT.f.terms[i].col_b = ucol_of(F.terms[i].col_b);
        }
        for (uint32_t i = 0; ok && i < FT.n_ucols; ++i) ok = ((uintptr_t)P.in[FT.ucol[i]].data & 15) == 0;
        const uint32_t smem = TMA_STAGES * FT.n_ucols * TMA_CHUNK * 8;
        if (ok && FT.n_ucols && smem <= (uint32_t)d->smem_optin - 4096) {
            FusedTmaParams *dFT = nullptr;
            int32_t rc2 = dalloc(r, &dFT, 1);
            if (rc2) return rc2;
            CU(cudaMemcpyAsync(dFT, &FT, sizeof(FT), cudaMemcpyHostToDevice, d->stream));
            const uint32_t sms = (uint32_t)d->prop.multiProcessorCount;
            switch (np) {
                case 1: rc2 = launch_fused_tma_np<1>(ntm, sms, P.n_tiles, smem, d->stream, dP, dFT); break;
                case 2: rc2 = launch_fused_tma_np<2>(ntm, sms, P.n_tiles, smem, d->stream, dP, dFT); break;
                case 3: rc2 = launch_fused_tma_np<3>(ntm, sms, P.n_tiles, smem, d->stream, dP, dFT); break;
                default: rc2 = launch_fused_tma_np<4>(ntm, sms, P.n_tiles, smem, d->stream, dP, dFT); break;
            }
            if (rc2) return rc2;
            CU(cudaGetLastError());
            r->launches += 1;
            return TPLX_OK;
        }
    }
    FusedParams *dF = nullptr;
    int32_t rc = dalloc(r, &dF, 1);
    if (rc) return rc;
    CU(cudaMemcpyAsync(dF, &F, sizeof(F), cudaMemcpyHostToDevice, d->stream));
    // memory-bound streaming kernel: fill every SM with resident CTAs (multiple of the SM count)
    const uint32_t grid = std::max<uint32_t>(1, std::min<uint32_t>(P.n_tiles, (uint32_t)d->prop.multiProcessorCount * 8));
    switch (np) {
        case 1: launch_fused_np<1>(ntm, grid, d->stream, dP, dF); break;
        case 2: launch_fused_np<2>(ntm, grid, d->stream, dP, dF); break;
        case 3: launch_fused_np<3>(ntm, grid, d->stream, dP, dF); break;
        case 4: launch_fused_np<4>(ntm, grid, d->stream, dP, dF); break;
        default: launch_fused_np<8>(ntm, grid, d->stream, dP, dF); break;
    }
    CU(cudaGetLastError());
    r->launches += 1;
    return TPLX_OK;
}

static int32_t run_agg(tplx_stage *s, StageDev *sd, const tplx_block *b, tplx_result *r) {
    Device *d = r->dev;
    const uint64_t n = b->n_rows;
    const uint32_t R = 16;
    // specialised K3 (jit.inl) for stages without a closed-form hint: compact register file = the accumulator inputs
    jit::Loaded *jf = nullptr;
    if (!(s->has_fused && !getenv("TPLX_NO_FUSED")) && jit_wanted(s, n))
        jf = jit_get(s, sd, jit::K_AGG, jit_minb(s, jit::K_AGG));
    Layout L = make_layout(s, R, false, false, jf != nullptr);
    if (L.total > (uint32_t)d->smem_optin) return fail(TPLX_E_UNSUPPORTED, "stage needs more shared memory than one SM has");
    int occ = 0;
    if (jf) occ = jit_occupancy(jf, L.total);
    else CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, stage_agg_kernel, NT, L.total));
    if (occ < 1) return fail(TPLX_E_UNSUPPORTED, "stage kernel cannot be resident");
    KParams P;
    fill_common(P, s, sd, b, L, R);
    if (jf) {
        P.n_instr = 0;
        P.n_slots = (uint32_t)s->jit_live.slots.size();
        for (size_t k = 0; k < s->accs.size(); ++k) P.accs[k].slot = (uint32_t)s->jit_live.map[s->accs[k].slot];
    }
    const uint32_t grid = std::max<uint32_t>(1, std::min<uint32_t>(P.n_tiles, (uint32_t)(occ * d->prop.multiProcessorCount)));
    P.scratch_per_thread = s->materialises ? std::max<uint32_t>(s->hdr.scratch_bytes, 64) : 0;
    int32_t rc = ensure_scratch(d, (size_t)grid * NT * P.scratch_per_thread);
    if (rc) return rc;
    P.scratch = d->scratch;
    uint64_t cap_exc = std::max<uint64_t>(4096, (uint64_t)(s->est_exc_per_row.load(relaxed) * 1.5 * (double)n) + n / 64);
    KParams *dP = nullptr;
    uint32_t *counters = nullptr;
    rc = dalloc(r, &P.tile_partials, (size_t)std::max<uint32_t>(P.n_tiles, 1) * P.n_accs);
    if (rc) return rc;
    rc = dalloc(r, &P.agg_out, TPLX_MAX_ACCS);
    if (rc) return rc;
    rc = dalloc(r, &counters, 4);
    if (rc) return rc;
    rc = dalloc(r, &dP, 1);
    if (rc) return rc;
    P.counters = counters;
    r->n_accs = P.n_accs;
    for (int attempt = 0; attempt < 2; ++attempt) {
        P.cap_exc = cap_exc;
        rc = dalloc(r, &P.exc, cap_exc);
        if (rc) return rc;
        CU(cudaMemsetAsync(counters, 0, 16, d->stream));
        CU(cudaMemcpyAsync(dP, &P, sizeof(P), cudaMemcpyHostToDevice, d->stream));
        CU(cudaEventRecord(r->evk0, d->stream));
        if (P.n_tiles && s->has_fused && !getenv("TPLX_NO_FUSED")) {
            int32_t frc = launch_fused(s, d, dP, P, r);
            if (frc) return frc;
        } else if (P.n_tiles && jf) {
            const KParams *dPc = dP;
            rc = jit_launch(jf, grid, L.total, d->stream, &dPc);
            if (rc) return rc;
            r->launches += 1;
            r->jit_launches += 1;
        } else if (P.n_tiles) {
            stage_agg_kernel<<<grid, NT, L.total, d->stream>>>(dP);
            CU(cudaGetLastError());
            r->launches += 1;
        }
        agg_finalize_kernel<<<1, FIN_NT, 0, d->stream>>>(dP);
        CU(cudaGetLastError());
        r->launches += 1;
        CU(cudaEventRecord(r->evk1, d->stream));
        uint32_t h_cnt[4];
        CU(cudaMemcpyAsync(h_cnt, counters, 16, cudaMemcpyDeviceToHost, d->stream));
        CU(cudaStreamSynchronize(d->stream));
        r->n_exc = h_cnt[2];
        if (n) s->est_exc_per_row.store((double)r->n_exc / (double)n, relaxed);
        if (!(h_cnt[1] & 4u)) break;
        cap_exc = r->n_exc + 16;
        if (attempt == 1) return fail(TPLX_E_OVERFLOW, "exception capacity retry failed");
    }
    r->agg_out = P.agg_out;
    r->exc = P.exc;
    r->n_out = 1;
    // exception records of an aggregate stage are appended in arbitrary order: sort by input row and
    // number them like TransformTask::_outputRowCounter would (no normal rows are written)
    if (r->n_exc) {
        std::vector<tplx_exception_rec> recs(r->n_exc);
        CU(cudaMemcpy(recs.data(), r->exc, r->n_exc * sizeof(tplx_exception_rec), cudaMemcpyDeviceToHost));
        std::sort(recs.begin(), recs.end(), [](const tplx_exception_rec &a, const tplx_exception_rec &b) { return a.row < b.row; });
        for (size_t i = 0; i < recs.size(); ++i) recs[i].row_no = (int64_t)i;
        CU(cudaMemcpy(r->exc, recs.data(), r->n_exc * sizeof(tplx_exception_rec), cudaMemcpyHostToDevice));
    }
    return TPLX_OK;
}

extern "C" int32_t tplx_gpu_result_info(tplx_result *r, tplx_result_info *info) {
    if (!r || !info) return fail(TPLX_E_BADARG, "result_info: bad arguments");
    CU(cudaSetDevice(r->dev->id));
    CU(cudaEventSynchronize(r->ev1));
    float ms = 0;
    CU(cudaEventElapsedTime(&ms, r->evk0, r->evk1));
    r->kernel_ms = ms + r->kernel_ms_extra;
    const bool trace = getenv("TPLX_TRACE") != nullptr;
    if (trace) fprintf(stderr, "[tplx] stage kernels %.3f ms, gather %.3f ms", ms, r->kernel_ms_extra);
    for (auto &e : r->extra_ev) {
        CU(cudaEventElapsedTime(&ms, e.first, e.second));
        r->kernel_ms += ms;
        if (trace) fprintf(stderr, ", prefilter %.3f ms", ms);
    }
    if (trace) fprintf(stderr, "\n");
    CU(cudaEventElapsedTime(&ms, r->ev0, r->ev1));
    r->total_ms = ms;
    memset(info, 0, sizeof(*info));
    info->n_in_rows = r->n_in;
    info->n_out_rows = r->n_out;
    info->n_exceptions = r->n_exc;
    for (size_t c = 0; c < r->str_bytes.size() && c < TPLX_MAX_COLS; ++c) info->out_str_bytes[c] = r->str_bytes[c];
    info->kernel_ms = r->kernel_ms;
    info->total_ms = r->total_ms;
    info->kernel_launches = r->launches;
    info->specialised_launches = r->jit_launches;
    info->lane = r->lane;
    info->zero_copy_cols = r->zero_copy_cols;
    info->h2d_bytes = r->h2d_bytes;
    return TPLX_OK;
}

extern "C" int32_t tplx_gpu_result_fetch_column(tplx_result *r, uint32_t col, void *data, uint32_t *offsets) {
    if (!r || col + r->hidden >= r->out.size()) return fail(TPLX_E_BADARG, "result_fetch_column: bad arguments");
    CU(cudaSetDevice(r->dev->id));
    const OutCol &oc = r->out[col];
    if (r->out_types[col] == TPLX_T_STR) {
        if (offsets) CU(cudaMemcpyAsync(offsets, oc.offsets, (r->n_out + 1) * 4, cudaMemcpyDeviceToHost, r->dev->d2h_stream));
        if (data && r->str_bytes[col]) CU(cudaMemcpyAsync(data, oc.bytes, r->str_bytes[col], cudaMemcpyDeviceToHost, r->dev->d2h_stream));
    } else if (data && r->n_out) {
        CU(cudaMemcpyAsync(data, oc.data, r->n_out * 8, cudaMemcpyDeviceToHost, r->dev->d2h_stream));
    }
    CU(cudaStreamSynchronize(r->dev->d2h_stream));
    return TPLX_OK;
}

extern "C" int32_t tplx_gpu_result_device_column(tplx_result *r, uint32_t col, const void **data, const uint32_t **offsets) {
    if (!r || col + r->hidden >= r->out.size()) return fail(TPLX_E_BADARG, "result_device_column: bad arguments");
    const OutCol &oc = r->out[col];
    if (r->out_types[col] == TPLX_T_STR) {
        if (data) *data = oc.bytes;
        if (offsets) *offsets = oc.offsets;
    } else {
        if (data) *data = oc.data;
        if (offsets) *offsets = nullptr;
    }
    return TPLX_OK;
}

extern "C" int32_t tplx_gpu_result_fetch_exceptions(tplx_result *r, tplx_exception_rec *recs) {
    if (!r || (!recs && r->n_exc)) return fail(TPLX_E_BADARG, "result_fetch_exceptions: bad arguments");
    if (!r->n_exc) return TPLX_OK;
    CU(cudaSetDevice(r->dev->id));
    CU(cudaMemcpyAsync(recs, r->exc, r->n_exc * sizeof(tplx_exception_rec), cudaMemcpyDeviceToHost, r->dev->d2h_stream));
    CU(cudaStreamSynchronize(r->dev->d2h_stream));
    return TPLX_OK;
}

extern "C" int32_t tplx_gpu_result_fetch_aggregate(tplx_result *r, int64_t *acc_bits) {
    if (!r || !acc_bits || !r->agg_out) return fail(TPLX_E_BADARG, "result_fetch_aggregate: not an aggregate result");
    CU(cudaSetDevice(r->dev->id));
    CU(cudaMemcpyAsync(acc_bits, r->agg_out, r->n_accs * 8, cudaMemcpyDeviceToHost, r->dev->d2h_stream));
    CU(cudaStreamSynchronize(r->dev->d2h_stream));
    return TPLX_OK;
}

#include "tplx_gpu_rowfmt.inl"
#include "tplx_gpu_hash.inl"
#include "tplx_gpu_csv.inl"
#include "tplx_gpu_text.inl"
#include "tplx_gpu_comm.inl"
#include "tplx_gpu_join.inl"
#include "tplx_gpu_merge.inl"
#include "tplx_gpu_concat.inl"
#include "tplx_gpu_sort.inl"
