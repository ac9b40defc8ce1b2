// ref_shim_segment stub (test infrastructure): the shim's tbb::parallel_for runs its body on the calling thread, so
// the reader-writer lock has nothing to exclude.
#pragma once
namespace tbb {
class spin_rw_mutex {
public:
    class scoped_lock {
    public:
        scoped_lock(spin_rw_mutex&, bool /*write*/) {}
        bool upgrade_to_writer() { return true; }
    };
};
}  // namespace tbb
