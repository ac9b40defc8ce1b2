"""``open3d.utility.random`` (pybind/utility/random.cpp): the library's process-global random engine, one
std::mt19937 in libo3db200.so that every random operation of the library draws from (utility/Random.cpp)."""
from .._lib import check, lib


def seed(seed):
    """Set the global random seed: the engine becomes std::mt19937(seed), as utility::random::Seed does.  Without a
    call the engine is seeded from std::random_device."""
    seed = int(seed)
    if not -2 ** 31 <= seed < 2 ** 31:
        # upstream's argument is a C int, which its binding refuses to take from a larger int
        raise TypeError(f"seed must fit in a 32-bit int (got {seed})")
    check(lib.o3db_random_seed(seed))
