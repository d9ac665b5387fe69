/* Minimal hand-written subset of Node's stable N-API (node_api.h is not present in this image).
 * Types and prototypes follow the published ABI-stable N-API v8 headers; when building inside a real
 * Node.js toolchain, define EB200_HAVE_NODE_API_H and `#include <node_api.h>` is used instead. */
#ifndef EB200_NODE_API_MIN_H
#define EB200_NODE_API_MIN_H
#include <stddef.h>
#include <stdint.h>
#include <stdbool.h>
typedef struct napi_env__* napi_env;
typedef struct napi_value__* napi_value;
typedef struct napi_ref__* napi_ref;
typedef struct napi_deferred__* napi_deferred;
typedef struct napi_async_work__* napi_async_work;
typedef struct napi_callback_info__* napi_callback_info;
typedef enum { napi_ok = 0 } napi_status;
typedef napi_value (*napi_callback)(napi_env env, napi_callback_info info);
typedef void (*napi_async_execute_callback)(napi_env env, void* data);
typedef void (*napi_async_complete_callback)(napi_env env, napi_status status, void* data);
typedef enum { napi_uint8_array = 1 } napi_typedarray_type;
#define NAPI_AUTO_LENGTH ((size_t)-1)
typedef struct {
  int nm_version; unsigned int nm_flags; const char* nm_filename;
  napi_value (*nm_register_func)(napi_env env, napi_value exports);
  const char* nm_modname; void* nm_priv; void* reserved[4];
} napi_module;
#ifdef __cplusplus
extern "C" {
#endif
void napi_module_register(napi_module* mod);
napi_status napi_get_cb_info(napi_env env, napi_callback_info cbinfo, size_t* argc, napi_value* argv, napi_value* this_arg, void** data);
napi_status napi_get_typedarray_info(napi_env env, napi_value typedarray, napi_typedarray_type* type, size_t* length, void** data, napi_value* arraybuffer, size_t* byte_offset);
napi_status napi_is_typedarray(napi_env env, napi_value value, bool* result);
napi_status napi_is_array(napi_env env, napi_value value, bool* result);
napi_status napi_get_array_length(napi_env env, napi_value value, uint32_t* result);
napi_status napi_get_element(napi_env env, napi_value object, uint32_t index, napi_value* result);
napi_status napi_get_value_uint32(napi_env env, napi_value value, uint32_t* result);
napi_status napi_get_value_int32(napi_env env, napi_value value, int32_t* result);
napi_status napi_create_arraybuffer(napi_env env, size_t byte_length, void** data, napi_value* result);
napi_status napi_create_typedarray(napi_env env, napi_typedarray_type type, size_t length, napi_value arraybuffer, size_t byte_offset, napi_value* result);
napi_status napi_create_object(napi_env env, napi_value* result);
typedef void (*napi_finalize)(napi_env env, void* finalize_data, void* finalize_hint);
napi_status napi_create_external(napi_env env, void* data, napi_finalize finalize_cb, void* finalize_hint, napi_value* result);
napi_status napi_get_value_external(napi_env env, napi_value value, void** result);
napi_status napi_create_uint32(napi_env env, uint32_t value, napi_value* result);
napi_status napi_create_double(napi_env env, double value, napi_value* result);
napi_status napi_create_function(napi_env env, const char* utf8name, size_t length, napi_callback cb, void* data, napi_value* result);
napi_status napi_set_named_property(napi_env env, napi_value object, const char* utf8name, napi_value value);
napi_status napi_throw_error(napi_env env, const char* code, const char* msg);
napi_status napi_get_undefined(napi_env env, napi_value* result);
napi_status napi_create_string_utf8(napi_env env, const char* str, size_t length, napi_value* result);
napi_status napi_create_error(napi_env env, napi_value code, napi_value msg, napi_value* result);
napi_status napi_create_reference(napi_env env, napi_value value, uint32_t initial_refcount, napi_ref* result);
napi_status napi_delete_reference(napi_env env, napi_ref ref);
napi_status napi_get_reference_value(napi_env env, napi_ref ref, napi_value* result);
napi_status napi_create_promise(napi_env env, napi_deferred* deferred, napi_value* promise);
napi_status napi_resolve_deferred(napi_env env, napi_deferred deferred, napi_value resolution);
napi_status napi_reject_deferred(napi_env env, napi_deferred deferred, napi_value rejection);
napi_status napi_create_async_work(napi_env env, napi_value async_resource, napi_value async_resource_name,
                                   napi_async_execute_callback execute, napi_async_complete_callback complete, void* data, napi_async_work* result);
napi_status napi_queue_async_work(napi_env env, napi_async_work work);
napi_status napi_delete_async_work(napi_env env, napi_async_work work);
#ifdef __cplusplus
}
#endif
#endif
