# nvcomp-config.cmake -- lets the reference's build system find this library:
#   cmake -S <nvCOMP tree> -B oracle/_ref/cmake -Dnvcomp_DIR=<this repo>/cmake -DBUILD_BENCHMARKS=ON
# satisfies `find_package(nvcomp 3.0.3 REQUIRED)` (reference CMakeLists.txt:18) and provides the imported target
# `nvcomp::nvcomp` the benchmarks/examples link (reference benchmarks/CMakeLists.txt:28;
# reference cmake/nvcomp-config.cmake.in:26,38).
get_filename_component(_NVCOMP_B200_ROOT "${CMAKE_CURRENT_LIST_DIR}/.." ABSOLUTE)
if(NOT TARGET nvcomp::nvcomp)
  add_library(nvcomp::nvcomp SHARED IMPORTED)
  set_target_properties(nvcomp::nvcomp PROPERTIES
    IMPORTED_LOCATION "${_NVCOMP_B200_ROOT}/nvcomp_b200/lib/libnvcomp.so"
    INTERFACE_INCLUDE_DIRECTORIES "${_NVCOMP_B200_ROOT}/include")
endif()
set(nvcomp_FOUND TRUE)
set(nvcomp_VERSION 3.0.3)
