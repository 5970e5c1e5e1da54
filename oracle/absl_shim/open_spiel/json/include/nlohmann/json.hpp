// TEST INFRASTRUCTURE ONLY: forwards to an nlohmann/json single header found on the include path (the reference expects
// it at open_spiel/json/, cloned by its install.sh).  oracle/ref_build.mk and open_spiel_b200/adapter/Makefile add the
// directory __graft_entry__.json_include_dir() finds as JSON_INC.
#pragma once
#include <nlohmann/json.hpp>
